"""Decode throughput at 8 and 16 cache rows per GPU (StarVector-1B dims, synthetic weights, greedy, EOS off).

    python scripts/batch_bench.py [--window 256] [--beam-steps 512] [--out results.json]

One call measures, with every shape warmed up first:
  (a) 8 rows on a max_batch=8 engine;
  (b) 16 rows on a max_batch=16 engine (two row groups sharing one weight stream);
  (c) 16 images as two sequential groups of 8 on the max_batch=8 engine (what the facade does above max_batch);
  (d) 8 images x 2 beams (16 rows) with the device beam search.
Per run: ms per decode step from sv_last_decode_timing (device events), tokens/s, and the HBM roofline fraction of the step
(bytes = decode weights + lm_head + KV read B * (L + 1) * kv_bytes_per_token at context L, over 3.35 TB/s) at a short and
a long context (the mean context of a 256-token window starting at ~300 and ~2300 positions).  The card's name and power
limit are printed in the same run.  Needs an H100.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from starvector_b200.beam_search import beam_search  # noqa: E402
from starvector_b200.config import dims_1b  # noqa: E402
from starvector_b200.engine import Engine, GenerationParams  # noqa: E402
from starvector_b200.weights import synthetic_images, synthetic_state_dict  # noqa: E402

HBM = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        q = f"nvidia-smi unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def step_bytes(d, rows, ctx):
    """Least HBM traffic of one decode step: every decoder weight and the lm_head once, plus each row's K/V over ctx + 1."""
    H, I, L, V = d.hidden, d.n_inner, d.n_layer, d.vocab
    qkv = H + 2 * d.n_kv_head * d.head_dim
    weights = 2 * L * (H * qkv + H * H + 2 * H * I) + 2 * V * H
    kv = 2 * 2 * L * d.n_kv_head * d.head_dim          # K and V, bf16, per row per token
    return weights + kv * rows * (ctx + 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--beam-steps", type=int, default=512)
    ap.add_argument("--window", type=int, default=256, help="decode steps per timed window")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("batch_bench needs a GPU")
    info = card()
    print(json.dumps(info), flush=True)
    d8 = dims_1b(max_batch=8, max_len=4096)
    sd = synthetic_state_dict(d8, seed=0, init="randomized")
    e8 = Engine(d8, 0); e8.load_state_dict(sd)
    d16 = dims_1b(max_batch=16, max_len=4096)
    e16 = Engine(d16, 0); e16.load_state_dict(sd)
    del sd
    img = synthetic_images(d8, 16, seed=1)
    Q = d8.query_length
    res = {"card": info, "engine16": e16.describe(), "runs": []}
    # each context: a 2-token prompt after the visual prefix, teacher-forced (scored) up to the target, then the timed window
    for label, target in (("ctx~300", 300), ("ctx~2300", 2300)):
        n = a.window
        extra = target - (Q + 2)
        shapes = {"a_8rows": (e8, [img[:8]]), "b_16rows": (e16, [img]), "c_2x8rows": (e8, [img[:8], img[8:]])}
        for rep in range(2):                                   # rep 0 warms every shape, rep 1 is reported
            for name, (eng, parts) in shapes.items():
                total_ms, total_steps = 0.0, 0
                for part in parts:
                    part = part.contiguous()
                    eng.encode_images(part)
                    eng.prefill(torch.full((part.shape[0], 2), 44, dtype=torch.int32))
                    eng.score(torch.full((part.shape[0], extra), 45, dtype=torch.int32, device="cuda"))
                    eng.generate(GenerationParams(max_new_tokens=n, eos_token_id=None, pad_token_id=0))
                    ms, steps = eng.last_decode_timing()
                    total_ms += ms
                    total_steps += steps
                if rep == 0:
                    continue
                rows = sum(p.shape[0] for p in parts)
                ctx = target + n // 2
                per_step = total_ms / total_steps * len(parts)          # one step = one token for every row
                byts = len(parts) * step_bytes(d8, rows // len(parts), ctx)
                r = {"shape": name, "context": label, "mean_ctx": ctx, "rows": rows, "steps": total_steps,
                     "ms_per_step": per_step, "tokens_per_s": rows * 1000.0 / per_step,
                     "hbm_roofline_fraction": byts / HBM / (per_step / 1000.0)}
                res["runs"].append(r)
                print(json.dumps(r), flush=True)
    # (d) 8 images x 2 beams, device beam search
    for rep in range(2):
        out = beam_search(e16, img[:8], torch.full((8, 2), 44, dtype=torch.int32), num_beams=2, max_new_tokens=a.beam_steps,
                          eos_token_id=None, pad_token_id=0, early_stopping="never", impl="device")
        ms, steps = e16.last_decode_timing()
        if rep:
            r = {"shape": "d_8x2beams", "rows": 16, "steps": steps, "ms_per_step": ms / steps,
                 "tokens_per_s": 8 * 1000.0 * steps / ms, "out_shape": list(out.shape)}
            res["runs"].append(r)
            print(json.dumps(r), flush=True)
    by = {(r["shape"], r.get("context")): r for r in res["runs"]}
    for ctx in ("ctx~300", "ctx~2300"):
        b, c = by[("b_16rows", ctx)], by[("c_2x8rows", ctx)]
        res[f"ratio_b_over_c_{ctx}"] = b["tokens_per_s"] / c["tokens_per_s"]
        print(f"{ctx}: 16 rows in one pass / two groups of 8 = {b['tokens_per_s'] / c['tokens_per_s']:.3f}", flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    e8.close(); e16.close()


if __name__ == "__main__":
    main()
