"""Continuous batching against groups of max_batch: useful tokens/s for a workload of ragged lengths.

    python scripts/continuous_bench.py [--images 64] [--rounds 2] [--out results.json]

StarVector-1B dims, synthetic weights, greedy decoding with EOS off, 16 cache rows.  The per-request token caps are
SYNTHETIC: a seeded lognormal (median 400 tokens, sigma 0.9) clipped to [64, 3000], standing in for the spread of SVG
lengths of a real dataset.  One call times two arms, alternated over `--rounds` rounds after one untimed warm-up round:
  (a) static: groups of 16 images through `Engine.generate`, each group run to its longest member (what a caller without
      continuous batching does);
  (b) continuous: `Engine.generate_requests` with 16 slots (a finished row is refilled with the next image at once).
Reported per arm and round: useful tokens/s (only the requested tokens count) from a host clock around synchronised
work, decode steps, and for (b) the share of the wall time spent in admission (encode + prefill).  The card's name and
power limit are read in the same call.  As an output check at the timed size, a sample of requests must equal a
one-image run at the session cap.  Needs an H100.
"""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from starvector_b200.config import dims_1b  # noqa: E402
from starvector_b200.continuous import ContinuousScheduler  # noqa: E402
from starvector_b200.engine import Engine, GenerationParams  # noqa: E402
from starvector_b200.weights import synthetic_images, synthetic_state_dict  # noqa: E402

SLOTS = 16
PROMPT = [44, 78]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        q = f"nvidia-smi unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def static_arm(eng, img, caps, params):
    steps = 0
    for lo in range(0, len(caps), SLOTS):
        n = max(caps[lo:lo + SLOTS])
        eng.encode_images(img[lo:lo + SLOTS])
        eng.prefill(torch.tensor([PROMPT] * min(SLOTS, len(caps) - lo)))
        eng.generate(dataclasses.replace(params, max_new_tokens=n))
        steps += n
    return steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--check", type=int, default=4, help="requests compared with a one-image run")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("continuous_bench needs a GPU")
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
    params = GenerationParams(max_new_tokens=cap, eos_token_id=None, pad_token_id=0)
    useful = sum(caps)
    res = {"card": info, "engine": eng.describe(), "images": a.images, "slots": SLOTS, "session_cap": cap,
           "caps_synthetic": {"dist": "lognormal(log 400, 0.9) clipped to [64, 3000]", "sum": useful,
                              "mean": useful / len(caps), "max": cap}, "rounds": []}
    print(json.dumps({k: res[k] for k in ("images", "slots", "session_cap", "caps_synthetic")}), flush=True)
    got = None
    for rnd in range(a.rounds + 1):                 # round 0 warms every graph shape and is not reported
        row = {"round": rnd}
        for arm in (("static", "continuous") if rnd % 2 == 0 else ("continuous", "static")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if arm == "static":
                steps = static_arm(eng, img, caps, params)
                extra = {}
            else:
                sch = ContinuousScheduler(eng, SLOTS)
                got = sch.run(img, torch.tensor(PROMPT), params, max_new_tokens=caps)
                steps = sch.stats["steps"]
                extra = {"admissions": sch.stats["admissions"], "admit_share": None, "admit_s": sch.stats["admit_s"]}
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            if arm == "continuous":
                extra["admit_share"] = extra["admit_s"] / wall
            row[arm] = {"wall_s": wall, "useful_tokens_per_s": useful / wall, "decode_steps": steps, **extra}
        if rnd:
            row["continuous_over_static"] = row["continuous"]["useful_tokens_per_s"] / row["static"]["useful_tokens_per_s"]
            res["rounds"].append(row)
        print(json.dumps(row), flush=True)
    assert [len(g) for g in got] == caps
    for k in np.linspace(0, a.images - 1, a.check).round().astype(int).tolist():      # output check at the timed size
        eng.encode_images(img[k:k + 1])
        eng.prefill(torch.tensor([PROMPT]))
        ref = eng.generate(params).cpu()[0][: caps[k]]
        assert torch.equal(got[k], ref), f"request {k} differs from its one-image run"
    res["output_check"] = f"{a.check} requests equal their one-image runs"
    r = [x["continuous_over_static"] for x in res["rounds"]]
    print(f"continuous / static useful tokens/s: {min(r):.3f} .. {max(r):.3f} over {len(r)} rounds; {res['output_check']}",
          flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
