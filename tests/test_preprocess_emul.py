"""Image preprocessing without a GPU (SURVEY.md §8f-2): the oracle restatement vs Pillow/torchvision, the library's
host-side pieces (resample taps, normalisation table, batch plan) vs the oracle, and the kernels' per-pixel arithmetic
(sv_preprocess_core.h, compiled for the host by a test harness) vs Pillow over the library's own batch plan."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import preprocess as P
from starvector_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [(224, 224, 3), (224, 224, 4), (64, 48, 4), (48, 64, 3), (1, 1, 3), (2, 5, 4), (300, 200, 4), (225, 223, 3),
         (640, 480, 3), (1000, 37, 3), (7, 900, 4), (512, 512, 4)]


class ImageMeta(C.Structure):                       # mirror of svpre::ImageMeta
    _fields_ = [("src_off", C.c_int64), ("tmp_off", C.c_int64)] + [(n, C.c_int32) for n in (
        "width", "height", "channels", "row_stride", "in_w", "in_h", "pad_left", "pad_top", "alpha_white", "kx_off", "ky_off",
        "ksize_x", "ksize_y")]


def _desc(size=224, alpha=_lib.SV_ALPHA_WHITE, pad=1, dtype=_lib.SV_DTYPE_F32, mean=P.CLIP_MEAN, std=P.CLIP_STD):
    return _lib.PreprocDesc(size, alpha, pad, dtype, (C.c_float * 3)(*mean), (C.c_float * 3)(*std))


@pytest.mark.parametrize("size", [224, 384])
def test_restatement_equals_pillow_and_torchvision(size):
    for i, (h, w, c) in enumerate(CASES):
        a = P.synthetic_image(h, w, c, seed=i)
        for alpha in (P.ALPHA_WHITE, P.ALPHA_DROP):
            ref, got = P.reference_transform(a, size, alpha), P.restated_transform(a, size, alpha)
            assert torch.equal(ref, got), (h, w, c, alpha)


def test_paste_on_white_exhaustive():
    from PIL import Image

    m, s = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    rgba = np.stack([s, 255 - s, (s * 7) % 256, m], axis=-1).astype(np.uint8)
    img = Image.fromarray(rgba, "RGBA")
    bg = Image.new("RGB", img.size, (255, 255, 255))
    bg.paste(img, mask=img.split()[3])
    assert np.array_equal(np.asarray(bg), P.paste_on_white(rgba))


def test_golden_fixture(golden_dir):
    g = torch.load(os.path.join(golden_dir, "preprocess_v1.pt"), weights_only=False)
    for case in g["cases"]:
        a = P.synthetic_image(*case["hwc"], seed=case["seed"])
        assert np.array_equal(a, case["image"].numpy())
        assert P.tensor_sha256(torch.from_numpy(P.restated_resized_u8(a, 224, case["alpha"]))) == case["resized_u8_sha256"]
        got = P.restated_transform(a, 224, case["alpha"])
        assert P.tensor_sha256(got) == case["sha256_f32"]
        assert P.tensor_sha256(got.to(torch.bfloat16)) == case["sha256_bf16"]


def test_siglip_restatement_and_golden(golden_dir):
    g = torch.load(os.path.join(golden_dir, "preprocess_v1.pt"), weights_only=False)
    for case in g["siglip_cases"]:
        a = P.synthetic_image(*case["hwc"], seed=case["seed"])
        ref, got = P.reference_siglip_transform(a, 384), P.restated_siglip_transform(a, 384)
        assert torch.equal(ref, got)
        assert P.tensor_sha256(got) == case["sha256_f32"] and P.tensor_sha256(got.to(torch.bfloat16)) == case["sha256_bf16"]


def test_library_taps_and_table_equal_oracle():
    lib = _lib.load()
    for out in (224, 384):
        for n in list(range(1, 34)) + [63, 223, 224, 225, 447, 448, 640, 1000, 1024, 4096, 16384]:
            ks = C.c_int32()
            assert lib.sv_resample_coeffs_host(n, out, C.byref(ks), None, None, 0) == 0
            b = np.zeros((out, 2), np.int32)
            t = np.zeros((out, ks.value), np.int32)
            ip = C.POINTER(C.c_int32)
            assert lib.sv_resample_coeffs_host(n, out, C.byref(ks), b.ctypes.data_as(ip), t.ctypes.data_as(ip), t.size) == 0
            k2, b2, t2 = P.precompute_coeffs(n, out)
            assert k2 == ks.value and np.array_equal(b, b2) and np.array_equal(t, t2), (n, out)
    lut = np.zeros((3, 256), np.float32)
    assert lib.sv_preproc_lut_host(C.byref(_desc()), lut.ctypes.data_as(C.POINTER(C.c_float))) == 0
    assert np.array_equal(lut.view(np.uint32), P.normalize_lut().view(np.uint32))
    half = (0.5, 0.5, 0.5)
    assert lib.sv_preproc_lut_host(C.byref(_desc(mean=half, std=half)), lut.ctypes.data_as(C.POINTER(C.c_float))) == 0
    assert np.array_equal(lut.view(np.uint32), P.normalize_lut(half, half).view(np.uint32))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("emul") / "preprocess_emul.so")
    subprocess.run([gxx, "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "emul", "preprocess_emul.cpp")],
                   check=True)
    lib = C.CDLL(so)
    lib.emul_preprocess.restype = C.c_int
    lib.emul_preprocess.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _run_emul(emul, arrays, desc):
    """plan (library, host) -> pack the input arena as sv_preproc_run_host's copies do -> both passes on the CPU."""
    lib = _lib.load()
    n = len(arrays)
    imgs = (_lib.ImageU8 * n)()
    keep = []
    for i, a in enumerate(arrays):
        keep.append(a)
        imgs[i] = _lib.ImageU8(a.ctypes.data, a.shape[1], a.shape[0], a.shape[2], a.strides[0] if a.strides[0] != a.shape[1] * a.shape[2] else 0)
    sizes = (C.c_int64 * 5)()
    assert lib.sv_preproc_plan_host(C.byref(desc), imgs, n, None, 0, sizes) == 0
    blob = np.zeros(sizes[0], np.uint8)
    assert lib.sv_preproc_plan_host(C.byref(desc), imgs, n, blob.ctypes.data, blob.size, sizes) == 0
    metas = (ImageMeta * n).from_buffer_copy(blob[: C.sizeof(ImageMeta) * n].tobytes())
    arena = np.full(sizes[2], 0xAB, np.uint8)                   # garbage between images must never be read
    for i, a in enumerate(arrays):
        m = metas[i]
        assert (m.width, m.height, m.channels, m.row_stride) == (a.shape[1], a.shape[0], a.shape[2], a.shape[1] * a.shape[2])
        tight = np.ascontiguousarray(a).reshape(-1)
        arena[m.src_off: m.src_off + tight.size] = tight
    S = desc.out_size
    tmp = np.zeros(sizes[3], np.uint32)
    out = np.zeros((n, S, S, 3), np.uint8)
    assert emul.emul_preprocess(arena.ctypes.data, blob.ctypes.data, sizes[1], n, S, tmp.ctypes.data, out.ctypes.data) == C.sizeof(ImageMeta)
    return out, metas, sizes


@pytest.mark.parametrize("alpha", [_lib.SV_ALPHA_WHITE, _lib.SV_ALPHA_DROP])
def test_kernel_arithmetic_equals_pillow_on_a_ragged_batch(emul, alpha):
    arrays = [P.synthetic_image(h, w, c, seed=10 + i) for i, (h, w, c) in enumerate(CASES)]
    wide = P.synthetic_image(90, 130, 4, seed=99)
    arrays.append(wide[:, 10:100])                              # a strided view: row_stride > width*channels
    out, metas, sizes = _run_emul(emul, arrays, _desc(alpha=alpha))
    for i, a in enumerate(arrays):
        ref = P.reference_resized_u8(np.ascontiguousarray(a), 224, alpha)
        assert np.array_equal(out[i], ref), (i, a.shape)
    assert sizes[4] == max(max(a.shape[:2]) for a in arrays)
    assert len({(m.kx_off, m.ksize_x) for m in metas}) < len(arrays)         # equal sizes share one coefficient table


def test_kernel_arithmetic_direct_resize_without_padding(emul):
    """pad_square = 0 (the SigLIP-style processor): (w,h) -> (S,S) with independent axis tables."""
    from PIL import Image

    arrays = [P.synthetic_image(h, w, 3, seed=40 + i) for i, (h, w) in enumerate([(300, 200), (100, 640), (384, 384), (17, 5)])]
    out, _, _ = _run_emul(emul, arrays, _desc(size=384, pad=0))
    for i, a in enumerate(arrays):
        ref = np.asarray(Image.fromarray(a, "RGB").resize((384, 384), Image.BICUBIC))
        assert np.array_equal(out[i], ref), (i, a.shape)


def test_plan_rejects_bad_images():
    lib = _lib.load()
    a = np.zeros((4, 4, 3), np.uint8)
    sizes = (C.c_int64 * 5)()
    for bad in (_lib.ImageU8(a.ctypes.data, 4, 4, 2, 0), _lib.ImageU8(a.ctypes.data, 0, 4, 3, 0), _lib.ImageU8(None, 4, 4, 3, 0),
                _lib.ImageU8(a.ctypes.data, 4, 4, 3, 5), _lib.ImageU8(a.ctypes.data, 20000, 4, 3, 0)):
        imgs = (_lib.ImageU8 * 1)(bad)
        assert lib.sv_preproc_plan_host(C.byref(_desc()), imgs, 1, None, 0, sizes) == _lib.SV_ERR_INVALID
        assert lib.sv_preproc_last_error(None)


def test_processor_fails_loudly_without_a_gpu():
    """No CPU fallback: on a machine without a usable sm_90 device the constructor raises (and says why)."""
    if torch.cuda.is_available():
        pytest.skip("needs a machine without a GPU")
    from starvector_b200.preprocess import ImageTrainProcessor, _as_u8_hwc

    with pytest.raises(_lib.EngineError, match="no CPU fallback"):
        ImageTrainProcessor(size=224)
    # host-side input validation does not need the device
    with pytest.raises(ValueError):
        _as_u8_hwc(np.zeros((4, 4), np.uint8))
    with pytest.raises(ValueError):
        _as_u8_hwc("not an image")
    view = np.zeros((8, 12, 4), np.uint8)[:, 2:9]
    assert _as_u8_hwc(view).strides == view.strides            # row-strided views are passed through, not copied
    assert _as_u8_hwc(np.zeros((8, 12, 4), np.uint8)[:, ::2]).flags["C_CONTIGUOUS"]      # pixel-strided ones are copied
