"""Beam sessions against groups of images through sv_beam_search: useful tokens/s for a workload of ragged lengths.

    python scripts/beam_session_bench.py [--images 64] [--rounds 2] [--out results.json]

StarVector-1B dims, synthetic weights, 2-beam search with EOS off, 16 cache rows (8 groups of 2 beams).  The per-request
token caps are SYNTHETIC, the seeded lognormal of continuous_bench.py (median 400 tokens, sigma 0.9, clipped to [64, 3000]).
One call times two arms, alternated over `--rounds` rounds after an untimed warm-up:
  (a) static: groups of 8 images through `sv_beam_search` (`beam_search(impl="device")`), each group run to its longest
      member (what a caller without beam sessions does);
  (b) session: `Engine.beam_requests` with 16 slots (a group whose search ended takes the next image at once).
Reported per arm and round: useful tokens/s (only the requested tokens count) from a host clock around synchronised
work, decode steps, and for (b) the share of the wall time spent in admission (encode + prefill + first step).  The card's
name and power limit are read in the same call.  As an output check at the timed size, requests whose cap gives the decode
attention the session cap's partition must equal their one-image searches.  Needs an H100.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from starvector_b200.beam_search import beam_search  # noqa: E402
from starvector_b200.config import dims_1b  # noqa: E402
from starvector_b200.continuous import ContinuousScheduler  # noqa: E402
from starvector_b200.engine import BeamSearchParams, Engine  # noqa: E402
from starvector_b200.weights import synthetic_images, synthetic_state_dict  # noqa: E402

SLOTS, NB = 16, 2
PROMPT = [44, 78]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        q = f"nvidia-smi unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def cluster_ctas(total_keys):
    """CTAs per image of the fused decode attention for a row of total_keys keys (attention_decode_cluster_ncta)."""
    return max(1, min(8, ((total_keys + 31) // 32 + 7) // 8))


def static_arm(eng, img, caps, kw):
    steps, per = 0, SLOTS // NB
    for lo in range(0, len(caps), per):
        n = max(caps[lo:lo + per])
        b = min(per, len(caps) - lo)
        beam_search(eng, img[lo:lo + per], torch.tensor([PROMPT] * b), max_new_tokens=n, impl="device", **kw)
        steps += n
    return steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--check", type=int, default=2, help="requests compared with a one-image search")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("beam_session_bench needs a GPU")
    info = card()
    print(json.dumps(info), flush=True)
    rng = np.random.default_rng(0)
    caps = [int(c) for c in np.clip(np.round(rng.lognormal(np.log(400.0), 0.9, a.images)), 64, 3000)]
    cap = max(caps)
    d = dims_1b(max_batch=SLOTS)
    d = dims_1b(max_batch=SLOTS, max_len=d.query_length + len(PROMPT) + cap + 64)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    eng = Engine(d, 0)
    eng.load_state_dict(sd)
    del sd
    img = synthetic_images(d, a.images, seed=1)
    kw = dict(num_beams=NB, eos_token_id=None, pad_token_id=0)       # beam_search's row fill without EOS: -1
    params = BeamSearchParams(NB, cap, eos_token_id=None, pad_token_id=-1)
    useful = sum(caps)
    res = {"card": info, "engine": eng.describe(), "images": a.images, "slots": SLOTS, "num_beams": NB, "session_cap": cap,
           "caps_synthetic": {"dist": "lognormal(log 400, 0.9) clipped to [64, 3000]", "sum": useful,
                              "mean": useful / len(caps), "max": cap}, "rounds": []}
    print(json.dumps({k: res[k] for k in ("images", "slots", "num_beams", "session_cap", "caps_synthetic")}), flush=True)
    # warm-up: both arms on the first 16 images at short caps (module loads, graph captures of the session shape)
    warm = [min(c, 64) for c in caps[:SLOTS]]
    static_arm(eng, img[:SLOTS], warm, kw)
    ContinuousScheduler(eng, SLOTS, num_beams=NB).run(img[:SLOTS], torch.tensor(PROMPT), params, max_new_tokens=warm)
    got = None
    for rnd in range(1, a.rounds + 1):
        row = {"round": rnd}
        for arm in (("static", "session") if rnd % 2 == 1 else ("session", "static")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if arm == "static":
                steps = static_arm(eng, img, caps, kw)
                extra = {}
            else:
                sch = ContinuousScheduler(eng, SLOTS, num_beams=NB)
                got = sch.run(img, torch.tensor(PROMPT), params, max_new_tokens=caps)
                steps = sch.stats["steps"]
                extra = {"admissions": sch.stats["admissions"], "admit_s": sch.stats["admit_s"]}
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            if arm == "session":
                extra["admit_share"] = extra["admit_s"] / wall
            row[arm] = {"wall_s": wall, "useful_tokens_per_s": useful / wall, "decode_steps": steps, **extra}
        row["session_over_static"] = row["session"]["useful_tokens_per_s"] / row["static"]["useful_tokens_per_s"]
        res["rounds"].append(row)
        print(json.dumps(row), flush=True)
    assert [len(g) for g in got] == caps                # no EOS: every search runs to its cap
    prefix = d.query_length + len(PROMPT)
    same = [k for k in range(a.images) if cluster_ctas(prefix + caps[k]) == cluster_ctas(prefix + cap)]
    for k in same[: a.check]:                           # output check at the timed size
        ref = beam_search(eng, img[k:k + 1], torch.tensor([PROMPT]), max_new_tokens=caps[k], impl="device", **kw).cpu()[0]
        assert torch.equal(got[k].long(), ref), f"request {k} differs from its one-image search"
    res["output_check"] = f"requests {same[:a.check]} equal their one-image searches"
    r = [x["session_over_static"] for x in res["rounds"]]
    print(f"session / static useful tokens/s: {min(r):.3f} .. {max(r):.3f} over {len(r)} rounds; {res['output_check']}",
          flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
