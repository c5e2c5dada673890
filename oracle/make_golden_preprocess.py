"""Writes tests/golden/preprocess_v1.pt: outputs of the reference's preprocessing recipe (oracle.preprocess
.reference_transform = Pillow 12.2 + torchvision 0.26, the reference's own dependencies, reference
starvector/data/util.py:40-66 / starvector_arch.py:39-45) on small deterministic images
(the resized bytes in full, the normalised fp32 / bf16 tensors as SHA-256 of their bytes to keep the fixture small).

    python -m oracle.make_golden_preprocess
"""
import os

import PIL
import torch
import torchvision

from oracle import preprocess as P

CASES = [((40, 56, 4), 1, P.ALPHA_WHITE), ((40, 56, 4), 1, P.ALPHA_DROP), ((300, 260, 3), 2, P.ALPHA_WHITE),
         ((9, 31, 4), 3, P.ALPHA_WHITE), ((224, 224, 3), 4, P.ALPHA_WHITE)]


def main():
    cases = []
    for hwc, seed, alpha in CASES:
        a = P.synthetic_image(*hwc, seed=seed)
        ref = P.reference_transform(a, 224, alpha)
        cases.append({"hwc": hwc, "seed": seed, "alpha": alpha, "image": torch.from_numpy(a),
                      "resized_u8_sha256": P.tensor_sha256(torch.from_numpy(P.reference_resized_u8(a, 224, alpha))),   # after Image.resize
                      "sha256_f32": P.tensor_sha256(ref), "sha256_bf16": P.tensor_sha256(ref.to(torch.bfloat16))})
    siglip = []
    for hwc, seed in [((50, 70, 4), 7), ((400, 300, 3), 8)]:
        a = P.synthetic_image(*hwc, seed=seed)
        ref = P.reference_siglip_transform(a, 384)
        siglip.append({"hwc": hwc, "seed": seed, "sha256_f32": P.tensor_sha256(ref), "sha256_bf16": P.tensor_sha256(ref.to(torch.bfloat16))})
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "preprocess_v1.pt")
    torch.save({"cases": cases, "siglip_cases": siglip, "versions": {"pillow": PIL.__version__, "torchvision": torchvision.__version__, "torch": torch.__version__}}, out)
    print(out, os.path.getsize(out))


if __name__ == "__main__":
    main()
