"""CPU oracle for image preprocessing (SURVEY.md §8f-2) — TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Two checkers for the same function, `uint8 HWC image -> float [3,S,S]`:

1. `reference_transform(img, ...)`: the reference's own recipe run with the reference's own dependencies, which ARE
   installed here and on the GPU box (Pillow 12.2, torchvision 0.26):
     * `ImageTrainProcessor` (reference starvector/data/util.py:40-66): RGBA -> paste on white with the alpha channel as
       mask (`:63-66`), pad to square with 255 (`:55-61`), `transforms.Resize(size, BICUBIC)` on the PIL image (`:49`,
       i.e. `Image.resize`, always antialiased), `ToTensor`, `Normalize(CLIP mean/std)` (`:33-38,50-51`);
     * `SimpleStarVectorProcessor` (reference starvector/model/starvector_arch.py:39-45): the same except RGBA is
       `convert("RGB")` (alpha dropped, `:40`).
   The recipe is restated here call for call (the reference module itself imports cairosvg/svgpathtools/bs4, which
   are not installed, so it cannot be imported).

2. `restated_transform(arr, ...)`: a numpy restatement of what those library calls compute, in the integer arithmetic
   of Pillow 12.2 (third-party dependency, not part of the reference; algorithm restated from its published source:
   `src/libImaging/Paste.c` `paste_mask_L` / `ImagingUtils.h` `MULDIV255`, `src/libImaging/Resample.c`
   `precompute_coeffs` / `normalize_coeffs_8bpc` / `ImagingResampleHorizontal_8bpc` / `ImagingResampleVertical_8bpc`,
   `bicubic_filter`).  This is the specification the CUDA kernels follow; it is pinned bit-for-bit to (1) in
   tests/test_preprocess_emul.py over a sweep of sizes, and (1) generated tests/golden/preprocess_v1.pt.
"""
from __future__ import annotations

import math
from typing import Sequence, Tuple

import numpy as np
import torch

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)          # data/util.py:33-36
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
PRECISION_BITS = 32 - 8 - 2                               # Resample.c: 8bpc fixed point

ALPHA_WHITE = 0     # ImageTrainProcessor._rgba_to_rgb_white
ALPHA_DROP = 1      # SimpleStarVectorProcessor: img.convert("RGB")


# ------------------------------------------------------------------------------------------------------------------
# (1) the reference recipe on the real libraries
def _to_pil(arr: np.ndarray):
    from PIL import Image

    assert arr.dtype == np.uint8 and arr.ndim == 3 and arr.shape[2] in (3, 4)
    return Image.fromarray(arr, "RGBA" if arr.shape[2] == 4 else "RGB")


def reference_transform(arr: np.ndarray, size: int = 224, alpha: int = ALPHA_WHITE, mean: Sequence[float] = CLIP_MEAN,
                        std: Sequence[float] = CLIP_STD) -> torch.Tensor:
    """float32 [3,size,size], exactly as the reference's processors build it."""
    from PIL import Image
    from torchvision import transforms
    from torchvision.transforms.functional import InterpolationMode, pad

    img = _to_pil(arr)
    if img.mode == "RGBA":
        if alpha == ALPHA_WHITE:                                         # data/util.py:63-66
            background = Image.new("RGB", img.size, (255, 255, 255))
            background.paste(img, mask=img.split()[3])
            img = background
        else:                                                            # starvector_arch.py:40
            img = img.convert("RGB")
    width, height = img.size                                             # data/util.py:55-61
    max_dim = max(width, height)
    padding = [(max_dim - width) // 2, (max_dim - height) // 2]
    padding += [max_dim - width - padding[0], max_dim - height - padding[1]]
    img = pad(img, padding, fill=255)
    img = transforms.Resize(size, interpolation=InterpolationMode.BICUBIC)(img)
    return transforms.Normalize(mean=mean, std=std)(transforms.ToTensor()(img))


def reference_siglip_transform(arr: np.ndarray, size: int = 384) -> torch.Tensor:
    """float32 [3,size,size] from the PIL-based SigLIP image processor of the installed transformers
    (`SiglipImageProcessorPil`: convert RGB, PIL bicubic resize to (size,size), x/255, mean = std = 0.5) — what
    `AutoProcessor.from_pretrained("google/siglip-*")` gave under the reference's pinned transformers 4.49
    (reference image_encoder.py:32-48, called at :119)."""
    import warnings

    from transformers.models.siglip import SiglipImageProcessorPil

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        proc = SiglipImageProcessorPil(size={"height": size, "width": size})
    return proc(images=_to_pil(arr), return_tensors="pt").pixel_values[0]


def restated_siglip_transform(arr: np.ndarray, size: int = 384) -> torch.Tensor:
    """numpy restatement of the above: alpha dropped, direct (w,h)->(size,size) resample, table normalisation."""
    u8 = resize_bicubic_u8(np.ascontiguousarray(arr[..., :3]), size, size)
    lut = normalize_lut((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))
    return torch.from_numpy(np.stack([lut[c][u8[..., c]] for c in range(3)]))


def reference_resized_u8(arr: np.ndarray, size: int = 224, alpha: int = ALPHA_WHITE) -> np.ndarray:
    """uint8 [size,size,3] right after the PIL resize (before ToTensor/Normalize)."""
    x = reference_transform(arr, size, alpha, mean=(0.0, 0.0, 0.0), std=(1.0, 1.0, 1.0))
    return (x * 255.0).round().to(torch.uint8).permute(1, 2, 0).numpy()


# ------------------------------------------------------------------------------------------------------------------
# (2) numpy restatement of the library arithmetic
def muldiv255(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """ImagingUtils.h MULDIV255: round(a*b/255) without a division."""
    tmp = a.astype(np.int32) * b.astype(np.int32) + 128
    return ((tmp >> 8) + tmp) >> 8


def paste_on_white(rgba: np.ndarray) -> np.ndarray:
    """Paste.c paste_mask_L with a 255 background: out = MULDIV255(255, 255-m) + MULDIV255(src, m)."""
    m = rgba[..., 3:4].astype(np.int32)
    out = muldiv255(np.full_like(m, 255), 255 - m) + muldiv255(rgba[..., :3], m)
    return out.astype(np.uint8)


def pad_to_square(rgb: np.ndarray) -> np.ndarray:
    h, w, _ = rgb.shape
    s = max(h, w)
    left, top = (s - w) // 2, (s - h) // 2
    out = np.full((s, s, 3), 255, np.uint8)
    out[top:top + h, left:left + w] = rgb
    return out


def bicubic_filter(x: float) -> float:
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def precompute_coeffs(in_size: int, out_size: int) -> Tuple[int, np.ndarray, np.ndarray]:
    """Resample.c precompute_coeffs + normalize_coeffs_8bpc for box (0, in_size): returns ksize,
    bounds int32 [out,2] = (first tap, tap count) and fixed-point taps int32 [out,ksize]."""
    scale = filterscale = float(in_size) / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = 2.0 * filterscale                       # bicubic support = 2
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    kk = np.zeros((out_size, ksize), np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = int(center - support + 0.5)
        if xmin < 0:
            xmin = 0
        xmax = int(center + support + 0.5)
        if xmax > in_size:
            xmax = in_size
        xmax -= xmin
        w = [bicubic_filter((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x in range(xmax):
            v = w[x] / ww if ww != 0.0 else w[x]
            kk[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return ksize, bounds, kk


def _clip8(ss: np.ndarray) -> np.ndarray:
    return np.clip(ss >> PRECISION_BITS, 0, 255).astype(np.uint8)


def resize_bicubic_u8(rgb: np.ndarray, out_w: int, out_h: int) -> np.ndarray:
    """`Image.resize((out_w,out_h), BICUBIC)` for an 8-bit RGB image: horizontal pass into an 8-bit
    intermediate, then vertical pass (Resample.c ImagingResampleInner)."""
    h, w, c = rgb.shape
    src = rgb.astype(np.int64)
    if w != out_w:
        _, bx, kx = precompute_coeffs(w, out_w)
        tmp = np.empty((h, out_w, c), np.uint8)
        for xx in range(out_w):
            x0, n = bx[xx]
            acc = (src[:, x0:x0 + n, :] * kx[xx, :n, None].astype(np.int64)[None]).sum(axis=1) + (1 << (PRECISION_BITS - 1))
            tmp[:, xx, :] = _clip8(acc)
        src = tmp.astype(np.int64)
    else:
        tmp = rgb
    if h != out_h:
        _, by, ky = precompute_coeffs(h, out_h)
        out = np.empty((out_h, out_w, c), np.uint8)
        for yy in range(out_h):
            y0, n = by[yy]
            acc = (src[y0:y0 + n] * ky[yy, :n, None, None].astype(np.int64)).sum(axis=0) + (1 << (PRECISION_BITS - 1))
            out[yy] = _clip8(acc)
        return out
    return np.ascontiguousarray(tmp)


def normalize_lut(mean: Sequence[float] = CLIP_MEAN, std: Sequence[float] = CLIP_STD) -> np.ndarray:
    """float32 [3,256]: ToTensor (`byte.to(float32).div(255)`) then Normalize (`sub_(mean).div_(std)`, fp32 tensors)
    evaluated for every byte value — the table the vertical-pass kernel looks up."""
    v = torch.arange(256, dtype=torch.uint8).to(torch.float32).div(255)
    m = torch.as_tensor(mean, dtype=torch.float32)
    s = torch.as_tensor(std, dtype=torch.float32)
    return ((v[None, :] - m[:, None]) / s[:, None]).numpy()


def restated_resized_u8(arr: np.ndarray, size: int = 224, alpha: int = ALPHA_WHITE) -> np.ndarray:
    rgb = arr[..., :3] if arr.shape[2] == 3 or alpha == ALPHA_DROP else paste_on_white(arr)
    return resize_bicubic_u8(pad_to_square(np.ascontiguousarray(rgb)), size, size)


def restated_transform(arr: np.ndarray, size: int = 224, alpha: int = ALPHA_WHITE, mean: Sequence[float] = CLIP_MEAN,
                       std: Sequence[float] = CLIP_STD) -> torch.Tensor:
    u8 = restated_resized_u8(arr, size, alpha)
    lut = normalize_lut(mean, std)
    out = np.stack([lut[c][u8[..., c]] for c in range(3)])
    return torch.from_numpy(out)


def tensor_sha256(t: torch.Tensor) -> str:
    import hashlib

    t = t.contiguous()
    raw = t.view(torch.int16) if t.dtype == torch.bfloat16 else t
    return hashlib.sha256(raw.numpy().tobytes()).hexdigest()


def synthetic_image(h: int, w: int, channels: int, seed: int) -> np.ndarray:
    """Deterministic test image: smooth gradients + hard edges + noise, with a structured alpha channel."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([(xx * 255 // max(w - 1, 1)), (yy * 255 // max(h - 1, 1)), ((xx + yy) * 7) % 256], axis=-1)
    noise = rng.integers(0, 256, size=(h, w, 3))
    mask = ((xx // 5 + yy // 3) % 2).astype(bool)[..., None]
    rgb = np.where(mask, base, noise).astype(np.uint8)
    if channels == 3:
        return rgb
    a = rng.integers(0, 256, size=(h, w, 1))
    a[: h // 3] = 255
    a[h - h // 4:] = 0
    return np.concatenate([rgb, a.astype(np.uint8)], axis=-1)
