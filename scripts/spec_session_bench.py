"""Speculative sessions against plain sessions (DESIGN.md §7i).

    python scripts/spec_session_bench.py [--rounds 2] [--out results.json]

StarVector-1B dims, synthetic weights, greedy decoding with EOS off.  Three measurements, each timing a plain and a
speculative session alternated over `--rounds` rounds after an untimed warm-up:
  1. full-load cost: 16 slots, all live, no spare column (so no drafts): device-event ms per verify step in a window of
     200 steps at ~400 and at ~2,400 keys of context.  This is the price every loaded session pays for speculation;
  2. the §7f workload: 64 requests with seeded lognormal caps (median 400, sigma 0.9, clipped to [64, 3000]) on 16 slots,
     plain against k = 3 and k = 7: useful tokens/s, verify steps, drafts proposed / accepted, outputs identical;
  3. light load: 2 requests of 1,024 tokens on 8 slots: per-request tokens/s, plain against k = 7.
The synthetic weights' greedy rows repeat, so almost every draft is accepted: 2 and 3 are UPPER BOUNDS of the gain, not a
measurement of it on real SVGs (the real checkpoint's acceptance is not measured here).  The card's name, power limit and
max SM clock are read in the same call.  Needs an H100.
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

PROMPT = [44, 78]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        q = f"nvidia-smi unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def full_load(eng, img, params, k, windows, n=200):
    """ms per step of a session of 16 live rows in each window (context reached before timing)."""
    p = dataclasses.replace(params, prompt_lookup_num_tokens=k)
    eng.session_begin(p, 16)
    out = {}
    try:
        eng.session_admit(img[:16], torch.tensor([PROMPT] * 16), list(range(16)))
        prefix = eng.query_length + len(PROMPT)
        done = 1
        for ctx in windows:
            ran, fin, _ = eng.session_run(ctx - prefix - done)
            done += ran
            assert not any(fin)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ran, fin, _ = eng.session_run(n)
            e1.record()
            torch.cuda.synchronize()
            assert ran == n and not any(fin)
            done += ran
            out[ctx] = e0.elapsed_time(e1) / n
        st = eng.session_spec_stats()
        if st is not None:
            assert st["drafted"] == 0
    finally:
        eng.session_end()
    return out


def workload(eng, img, params, k, caps, slots):
    sch = ContinuousScheduler(eng, slots)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    got = sch.run(img, torch.tensor(PROMPT), dataclasses.replace(params, prompt_lookup_num_tokens=k), max_new_tokens=caps)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return got, {"wall_s": wall, "useful_tokens_per_s": sum(caps) / wall, "verify_steps": sch.stats["steps"],
                 **(sch.stats.get("spec") or {})}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--images", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("spec_session_bench needs a GPU")
    info = card()
    print(json.dumps(info), flush=True)
    rng = np.random.default_rng(0)
    caps = [int(c) for c in np.clip(np.round(rng.lognormal(np.log(400.0), 0.9, a.images)), 64, 3000)]
    d = dims_1b(max_batch=16, max_len=4096)
    eng = Engine(d, 0)
    eng.load_state_dict(synthetic_state_dict(d, seed=0, init="randomized"))
    img = synthetic_images(d, a.images, seed=1)
    params = GenerationParams(max_new_tokens=3000, eos_token_id=None, pad_token_id=0)
    res = {"card": info, "engine": eng.describe(), "synthetic_weights_upper_bound": True, "full_load": [], "workload": [],
           "light": []}
    windows = [400, 2400]
    fl_params = dataclasses.replace(params, max_new_tokens=2700)
    for rnd in range(a.rounds + 1):              # round 0 warms every graph shape and is not reported
        arms = (0, 15) if rnd % 2 == 0 else (15, 0)
        row = {"round": rnd}
        for k in arms:
            row["spec_k15" if k else "plain"] = full_load(eng, img, fl_params, k, windows, n=200 if rnd else 20)
        row["spec_over_plain"] = {c: row["spec_k15"][c] / row["plain"][c] for c in windows}
        print(json.dumps({"full_load_ms_per_step": row}), flush=True)
        if rnd:
            res["full_load"].append(row)
    for rnd in range(a.rounds + 1):
        ks = (0, 3, 7) if rnd % 2 == 0 else (7, 3, 0)
        row, outs = {"round": rnd}, {}
        for k in ks:
            outs[k], row[f"k{k}"] = workload(eng, img if rnd else img[:16], params, k, caps if rnd else caps[:16], 16)
        assert all(len(outs[0]) == len(outs[k]) and all(torch.equal(x, y) for x, y in zip(outs[0], outs[k])) for k in ks)
        row["identical"] = True
        print(json.dumps({"workload": row}), flush=True)
        if rnd:
            res["workload"].append(row)
    for rnd in range(a.rounds + 1):
        ks = (0, 7) if rnd % 2 == 0 else (7, 0)
        row, outs = {"round": rnd}, {}
        n = 1024 if rnd else 64
        for k in ks:
            outs[k], r = workload(eng, img[:2], dataclasses.replace(params, max_new_tokens=n), k, [n, n], 8)
            r["per_request_tokens_per_s"] = n / r["wall_s"]
            row[f"k{k}"] = r
        assert all(torch.equal(x, y) for x, y in zip(outs[0], outs[7]))
        print(json.dumps({"light": row}), flush=True)
        if rnd:
            res["light"].append(row)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
