"""Generate tests/golden/*.pt by running the REFERENCE's own modules in this container.

Run from the repo root with a checkout of the reference:
    STARVECTOR_REF=<path to joanrod/star-vector> python -m oracle.make_golden

What is reference code here: ``VisionTransformer`` / ``LayerNorm``
(starvector/model/image_encoder/clip_model.py) and ``Adapter``
(starvector/model/adapters/adapter.py), imported in place through `oracle/ref_shim.py`,
plus the installed ``transformers`` GPTBigCode + ``generate`` that the reference calls.
``StarVectorBase`` itself cannot be constructed offline (needs omegaconf, hub access —
SURVEY.md §8c), so the glue between those modules is the restatement in
`oracle/pipeline.py`; the fixtures pin that restatement's vision/adapter half bit-for-bit
to the reference modules and record the decoder outputs for regression.
"""
from __future__ import annotations

import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import ref_shim  # noqa: E402
from oracle.pipeline import OracleStarVector, OracleStarVectorV2, VIS, LNV, ADP  # noqa: E402
from starvector_b200.config import dims_tiny, dims_tiny_v2  # noqa: E402
from starvector_b200.weights import synthetic_state_dict, synthetic_images  # noqa: E402

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
PROMPT_IDS = [44, 78]
STOP_IDS = [5, 6, 7]


def reference_vision(d, sd, img, adapter_norm):
    VT, LN, AD = ref_shim.load()
    vt = VT(d.image_size, d.patch_size, d.vit_width, d.vit_layers, d.vit_heads, False)
    vt.load_state_dict({k[len(VIS):]: v for k, v in sd.items() if k.startswith(VIS)})
    ln = LN(d.vit_width)
    ln.load_state_dict({k[len(LNV):]: v for k, v in sd.items() if k.startswith(LNV)})
    ad = AD(d.vit_width, d.hidden, adapter_norm=adapter_norm, query_length=d.query_length)
    ad.load_state_dict({k[len(ADP):]: v for k, v in sd.items() if k.startswith(ADP)}, strict=False)
    vt, ln, ad = vt.to(torch.bfloat16).eval(), ln.to(torch.bfloat16).eval(), ad.to(torch.bfloat16).eval()
    with torch.no_grad():
        v = ln(vt(img))
        return v, ad(v)


def main() -> None:
    torch.manual_seed(0)
    torch.set_num_threads(1)          # fixed reduction order for reproducible bits
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    for norm_id, norm in ((0, "layer_norm"), (1, "batch_norm")):
        d = dims_tiny(adapter_norm=norm_id)
        sd = synthetic_state_dict(d, seed=0, init="randomized")
        img = synthetic_images(d, 2, seed=1)
        vit_out, adapter_out = reference_vision(d, sd, img, norm)
        out = {"dims": d.__dict__.copy(), "seed": 0, "init": "randomized", "image_seed": 1,
               "prompt_ids": PROMPT_IDS, "stop_ids": STOP_IDS,
               "vit_out": vit_out, "adapter_out": adapter_out}
        if norm_id == 0:
            pad = d.vocab - 4
            for tag, dt in (("bf16", torch.bfloat16), ("fp32", torch.float32)):
                o = OracleStarVector(d, sd, dtype=dt, pad_token_id=pad)
                n_new = 24
                ids, logits = o.generate_im2svg_ids(
                    img, PROMPT_IDS, STOP_IDS, return_logits=True, use_nucleus_sampling=False, num_beams=1,
                    max_length=d.query_length + len(PROMPT_IDS) + n_new)
                g = torch.Generator().manual_seed(7)
                forced = torch.randint(1, d.vocab - 4, (2, n_new), generator=g)
                out[f"greedy_ids_{tag}"] = ids
                out[f"greedy_logits_{tag}"] = logits
                out["forced_ids"] = forced
                out[f"tf_logits_{tag}"] = o.teacher_forced_logits(img, PROMPT_IDS, forced)
        path = os.path.join(GOLDEN_DIR, f"tiny_v1_{norm}.pt")
        torch.save(out, path)
        print("wrote", path, os.path.getsize(path) // 1024, "KiB")
    # v2 (8B family): both towers are third-party transformers classes the reference loads by name; the reference's
    # own Adapter module is run on the SigLIP output.  40 new tokens cross the tiny config's 24-token sliding window.
    d = dims_tiny_v2()
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    img = synthetic_images(d, 2, seed=1)
    out = {"dims": d.__dict__.copy(), "seed": 0, "init": "randomized", "image_seed": 1, "prompt_ids": PROMPT_IDS,
           "stop_ids": STOP_IDS}
    _, _, AD = ref_shim.load()
    for tag, dt in (("bf16", torch.bfloat16), ("fp32", torch.float32)):
        o = OracleStarVectorV2(d, sd, dtype=dt)
        n_new = 40
        vit = o.image_encoder(img.to(dt))
        ad = AD(d.vit_width, d.hidden, adapter_norm="layer_norm", query_length=d.query_length)
        ad.load_state_dict({k[len(ADP):]: v for k, v in sd.items() if k.startswith(ADP)})
        ad = ad.to(dt).eval()
        with torch.no_grad():
            out[f"vit_out_{tag}"], out[f"adapter_out_{tag}"] = vit, ad(vit)
        ids, logits = o.generate_im2svg_ids(img, PROMPT_IDS, STOP_IDS, return_logits=True, use_nucleus_sampling=False,
                                            num_beams=1, max_length=d.query_length + len(PROMPT_IDS) + n_new)
        g = torch.Generator().manual_seed(7)
        forced = torch.randint(1, d.vocab - 5, (2, n_new), generator=g)
        out[f"greedy_ids_{tag}"], out[f"greedy_logits_{tag}"], out["forced_ids"] = ids, logits, forced
        out[f"tf_logits_{tag}"] = o.teacher_forced_logits(img, PROMPT_IDS, forced)
    path = os.path.join(GOLDEN_DIR, "tiny_v2_layer_norm.pt")
    torch.save(out, path)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
