"""Short 1B run for a profiler: encode + prefill + a few decode steps."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from starvector_b200.config import dims_1b
from starvector_b200.engine import Engine, GenerationParams
from starvector_b200.weights import synthetic_images, synthetic_state_dict

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=1)
ap.add_argument("--new", type=int, default=6)
ap.add_argument("--ctx", type=int, default=0, help="teacher-force this many tokens first to profile at a long context")
ap.add_argument("--reps", type=int, default=2)
a = ap.parse_args()
d = dims_1b(max_batch=a.batch, max_len=min(8192, 300 + a.ctx + a.new + 64))
eng = Engine(d, 0)
eng.load_state_dict(synthetic_state_dict(d, seed=0))
img = synthetic_images(d, a.batch, seed=1).cuda()
prompt = torch.tensor([[44, 5678]] * a.batch, dtype=torch.int32).cuda()
for rep in range(a.reps):
    eng.encode_images(img)
    eng.prefill(prompt)
    ids = eng.generate(GenerationParams(max_new_tokens=a.ctx + a.new, eos_token_id=None, pad_token_id=49152))
    torch.cuda.synchronize()
    ms, steps = eng.last_decode_timing()
    print(f"rep {rep}: {steps} decode steps in {ms:.3f} ms -> {ms / max(steps, 1) * 1000:.1f} us/step", flush=True)
if os.environ.get("SV_MEGA_DEBUG"):
    tl = eng.debug_timeline()
    if tl:
        t0 = tl[0]
        names = ["qkv", "attn_part", "attn_merge", "c_proj", "fc", "proj"]
        work = [(tl[i] - (tl[i - 1] if i else t0)) for i in range(0, len(tl), 2)]      # compute before barrier k
        bar = [(tl[i + 1] - tl[i]) for i in range(0, len(tl) - 1, 2)]                  # time inside barrier k
        print("stamps", len(tl), "total cycles", tl[-1] - t0)
        for k in range(0, min(len(bar), 12)):
            print(f"  phase {k:3d} {names[k % 6]:10s} work {work[k]:7d} cyc   barrier {bar[k]:7d} cyc")
        per = {n: [0, 0] for n in names}
        for k in range(min(len(bar), 144)):
            per[names[k % 6]][0] += work[k]; per[names[k % 6]][1] += bar[k]
        for n, (w, b) in per.items():
            print(f"  sum over 24 layers {n:10s} work {w:9d} cyc  barrier {b:9d} cyc")
        print("  tail (lm_head, select):", [(work[k], bar[k]) for k in range(144, len(bar))])
eng.close()
