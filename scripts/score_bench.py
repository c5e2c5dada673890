"""Teacher-forced scoring probe (not the headline bench): `sv_score_tokens` on the GRPO shape, StarVector-1B, one image
prefilled once, `expand_batch` to 8 rows, 4096 scored tokens per row.  Reports scored tokens/s and ms per call from CUDA
events, achieved TFLOP/s from algorithmic FLOPs and their share of the 989 TFLOP/s bf16 data-sheet rate (with the card's
name and power limit read in the same run), the per-token `forward()` path's time on the first 256 tokens and whether
both paths' log-probs agree.  One JSON line."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def run_score(args, G: int = 8, T: int = 4096, n_check: int = 256):
    """`sv_score_tokens` on the GRPO shape.  Times the chunked path with CUDA events, computes achieved TFLOP/s from
    algorithmic FLOPs (per token: 2 * (decoder params + V * H) for the matmuls, 4 * n_head * D * ctx per layer for attention,
    ctx = the token's cache length), and on the first `n_check` tokens times the per-token `forward()` path and checks that
    both paths' log-probs agree."""
    from starvector_b200.config import dims_1b
    from starvector_b200.engine import Engine
    from starvector_b200.weights import synthetic_state_dict

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    d = dims_1b(max_batch=G, max_len=T + 512)
    eng = Engine(d, 0)
    eng.load_state_dict(synthetic_state_dict(d, seed=0, device=dev))
    g = torch.Generator().manual_seed(0)
    prefix = (torch.randn(1, d.query_length, d.hidden, generator=g) * 0.5).to(torch.bfloat16).to(dev)
    ids = torch.randint(0, d.vocab, (G, T), generator=g).to(dev)

    def prep():
        first = eng.prefill_embeds(prefix, return_logits=True)
        eng.expand_batch([0] * G)
        return first

    def timed(fn):
        prep()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        out = fn()
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1), out

    for _ in range(max(1, args.warmup)):
        timed(lambda: eng.score(ids))
    ms = []
    for _ in range(max(1, args.steps)):
        t, lp = timed(lambda: eng.score(ids))
        ms.append(t)
    ms_call = sorted(ms)[len(ms) // 2]

    # the per-token path StarVectorForCausalLM.forward runs (one sv_decode_step per completion token), on the first n_check tokens
    first = prep()
    ref = torch.empty(G, n_check, device=dev)
    prev = first.repeat(G, 1)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for t in range(n_check):
        ref[:, t] = torch.log_softmax(prev, dim=-1).gather(-1, ids[:, t:t + 1].long()).squeeze(-1)
        prev = eng.decode_step(ids[:, t])
    t1.record()
    torch.cuda.synchronize()
    ms_tok_decode = t0.elapsed_time(t1) / n_check
    err = (lp[:, :n_check] - ref).abs()
    tol_max, tol_mean = 0.25, 0.03          # the bf16 bound tests/test_full_1b_gpu.py holds the decode path to
    agree = bool(err.max().item() < tol_max and err.mean().item() < tol_mean)

    H, L, V, I, q0 = d.hidden, d.n_layer, d.vocab, d.n_inner, d.query_length
    kv = d.n_kv_head * d.head_dim
    params = L * (H * (H + 2 * kv) + H * H + 2 * H * I)
    ctx_sum = sum(q0 + t + 1 for t in range(T))                 # keys each scored token attends to
    flops = G * (T * 2 * (params + V * H) + L * 4 * d.n_head * d.head_dim * ctx_sum)
    tflops = flops / (ms_call * 1e-3) / 1e12
    smi = {}
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().split(", ")
        smi = {"name": out[0], "power_limit": out[1], "sm_max_clock": out[2]}
    except Exception as e:                                        # noqa: BLE001 - the card name then comes from torch only
        smi = {"name": torch.cuda.get_device_name(0), "error": str(e)[:200]}
    line = {
        "metric": "teacher-forced scoring throughput", "value": G * T / (ms_call * 1e-3), "unit": "scored tokens/s",
        "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "dtype": "bf16",
        "data": "synthetic (random-init StarVector-1B weights, seeded prefix embeddings and token ids)",
        "config": {"workload": f"StarVector-1B, 1 image ({q0}-token prefix) prefilled once, expand_batch to {G} rows, "
                               f"{T} scored tokens per row (sv_score_tokens)"},
        "ms_per_call": ms_call, "ms_per_call_all": ms,
        "achieved_tflops": tflops, "algorithmic_tflop_per_call": flops / 1e12,
        "bf16_datasheet_tflops": 989.0, "frac_of_datasheet": tflops / 989.0,
        "gpu": smi,
        "per_token_path": {"ms_per_token": ms_tok_decode, "tokens_timed": n_check,
                           "ms_per_call_extrapolated": ms_tok_decode * T,
                           "speedup": ms_tok_decode * T / ms_call},
        "parity": {"tokens": n_check, "max_abs_diff": err.max().item(), "mean_abs_diff": err.mean().item(),
                   "tol_max": tol_max, "tol_mean": tol_mean, "agree": agree},
    }
    print(json.dumps(line), flush=True)
    eng.close()
    if not agree:
        raise SystemExit("score_bench: the chunked and per-token log-probs disagree")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    run_score(ap.parse_args())


if __name__ == "__main__":
    main()
