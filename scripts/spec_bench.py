"""Prompt-lookup speculative decoding at batch one (StarVector-1B dims, synthetic weights, greedy, EOS off).

    python scripts/spec_bench.py [--window 128] [--new 512] [--out results.json]

One call measures, with every shape warmed up first:
  (1) the cost curve: ms per verify step against k + 1 in {1, 2, 4, 8, 16} columns (k + 1 = 1 is the plain decode step)
      at contexts of ~400 and ~2400 tokens (a 2-token prompt after the visual prefix, teacher-forced up to the target,
      then a `--window`-token generation).  Per step = sv_last_decode_timing (device events around the replay loop, so
      the speculative loop's host polls are included) over the replays it ran.  Every replay verifies k + 1 columns
      whatever is accepted, so the synthetic weights' acceptance does not enter this number;
  (2) end to end: decode-loop tokens/s of plain against k = 3 and k = 7, alternating in one call, two runs each, with the
      outputs compared bit for bit.  The acceptance printed is a property of the synthetic weights, not of StarVector;
  (3) from (1), the break-even acceptance per k: the accepted drafts per verify step needed to beat plain decoding,
      T(k + 1) / T(1) - 1.
The card's name and power limit are printed in the same run.  Needs an H100.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from starvector_b200.config import dims_1b  # noqa: E402
from starvector_b200.engine import Engine, GenerationParams  # noqa: E402
from starvector_b200.weights import synthetic_images, synthetic_state_dict  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        q = f"nvidia-smi unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def run(eng, img, n_new, k, extra=0):
    eng.encode_images(img)
    eng.prefill(torch.full((1, 2), 44, dtype=torch.int32))
    if extra > 0:
        eng.score(torch.full((1, extra), 45, dtype=torch.int32, device="cuda"))
    out = eng.generate(GenerationParams(max_new_tokens=n_new, eos_token_id=None, pad_token_id=0, prompt_lookup_num_tokens=k))
    ms, steps = eng.last_decode_timing()
    return out.cpu(), ms, steps, (eng.last_spec_stats() if k else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window", type=int, default=128, help="tokens generated per cost-curve measurement")
    ap.add_argument("--new", type=int, default=512, help="tokens generated per end-to-end run")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("spec_bench needs a GPU")
    info = card()
    print(json.dumps(info), flush=True)
    d = dims_1b(max_batch=16, max_len=4096)
    eng = Engine(d, 0)
    eng.load_state_dict(synthetic_state_dict(d, seed=0, init="randomized"))
    img = synthetic_images(d, 1, seed=1)
    Q = d.query_length
    res = {"card": info, "engine": eng.describe(), "curve": [], "e2e": []}

    # (1) cost curve
    for label, target in (("ctx~400", 400), ("ctx~2400", 2400)):
        for rep in range(2):                                   # rep 0 warms every shape, rep 1 is reported
            for cols in (1, 2, 4, 8, 16):
                _, ms, steps, st = run(eng, img, a.window, cols - 1, extra=target - (Q + 2))
                if rep == 0:
                    continue
                r = {"context": label, "columns": cols, "replays": steps, "ms_per_step": ms / steps,
                     "tokens_per_step": a.window / steps if cols > 1 else 1.0}
                res["curve"].append(r)
                print(json.dumps(r), flush=True)
    by = {(r["context"], r["columns"]): r["ms_per_step"] for r in res["curve"]}
    for label in ("ctx~400", "ctx~2400"):
        t1 = by[(label, 1)]
        for cols in (2, 4, 8, 16):
            be = {"context": label, "k": cols - 1, "verify_over_plain": by[(label, cols)] / t1,
                  "break_even_accepted_per_step": by[(label, cols)] / t1 - 1.0}
            res.setdefault("break_even", []).append(be)
            print(json.dumps(be), flush=True)

    # (2) end to end, alternating plain / k = 3 / k = 7, two runs each after a warm-up round
    for rnd in range(3):
        ref = None
        for k in (0, 3, 7):
            out, ms, steps, st = run(eng, img, a.new, k)
            if ref is None:
                ref = out
            same = bool(torch.equal(out, ref))
            if rnd == 0:
                continue
            r = {"run": rnd, "k": k, "tokens": out.shape[1], "decode_ms": ms, "replays": steps,
                 "tokens_per_s": out.shape[1] * 1000.0 / ms, "equal_to_plain": same,
                 "synthetic_weights_acceptance": st}
            res["e2e"].append(r)
            print(json.dumps(r), flush=True)
            assert same, "speculative output differs from plain decoding"
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
