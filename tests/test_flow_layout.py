"""The flagged word layout of the dataflow decode kernel's exchange buffers (sv_decode_flow.cu, sv_op_decode_flow), decoded on
the CPU from the documented format, and the decoder checked against hand-built buffers.

* a flagged bf16 word: value in the low 16 bits, phase tag in the high 16; the tag of phase gp is (gp & 0x7fff) + 1;
* word i of a row sits at (i >> 3) * 64 + (i & 7): the 8 words of a fragment are contiguous, fragments 256 bytes apart;
  rows are (n >> 3) * 64 words apart;
* an attention partial word is 64 bits: fp32 value low, tag gp + 1 high; the partial of (row b, kv head h, item c) is
  PSZ = 32 + 16 * 128 words at ((b * n_kv + h) * MAXS + c) * PSZ: m[16], l[16], acc[16][128];
* an lm_head argmax partial (tile t, row b) is the 64-bit word t * 8 + b: [tag16 | bf16 value | index].
"""
import numpy as np
import torch

FRAG_STRIDE = 64
MAXS = 64
D = 128
PSZ = 32 + 16 * D


def tag16(gp):
    return ((gp & 0x7FFF) + 1)


def tag32(gp):
    return (gp + 1) & 0xFFFFFFFF


def row_words(n):
    return (n >> 3) * FRAG_STRIDE


def word_index(n):
    i = np.arange(n)
    return (i >> 3) * FRAG_STRIDE + (i & 7)


def _u32(words):
    return words.detach().cpu().numpy().view(np.uint32)


def _u64(words):
    return words.detach().cpu().numpy().view(np.uint64)


def decode_rows(words, B, n):
    """int32 flagged words -> (bf16 values [B, n], tags [B, n] int64)."""
    w = np.ascontiguousarray(_u32(words)[:B * row_words(n)].reshape(B, row_words(n))[:, word_index(n)])
    vals = torch.from_numpy((w & 0xFFFF).astype(np.uint16).view(np.int16)).view(torch.bfloat16)
    return vals, torch.from_numpy((w >> 16).astype(np.int64))


def decode_partial(words, b, h, c, n_kv):
    """int64 partial words of (row b, kv head h, item c) -> (m [16], l [16], acc [16, 128]) fp32 and their tags."""
    base = ((b * n_kv + h) * MAXS + c) * PSZ
    w = _u64(words)[base:base + PSZ]
    vals = torch.from_numpy((w & np.uint64(0xFFFFFFFF)).astype(np.uint32).view(np.float32))
    tags = torch.from_numpy((w >> np.uint64(32)).astype(np.int64))
    return (vals[:16], vals[16:32], vals[32:].view(16, D)), tags


def decode_amax(words, ntiles, B):
    """int64 argmax partial words -> (tag16 [ntiles, B], bf16 value [ntiles, B], index [ntiles, B])."""
    w = np.ascontiguousarray(_u64(words)[:ntiles * 8].reshape(ntiles, 8)[:, :B])
    tags = torch.from_numpy((w >> np.uint64(48)).astype(np.int64))
    vals = torch.from_numpy(((w >> np.uint64(32)) & np.uint64(0xFFFF)).astype(np.uint16).view(np.int16)).view(torch.bfloat16)
    idx = torch.from_numpy((w & np.uint64(0xFFFFFFFF)).astype(np.int64))
    return tags, vals, idx


def plan(N, ncta):
    """(rows per tile R, tiles) of a [N][K] GEMV over ncta CTAs (sv_ring.cuh make_plan)."""
    rpc = (N + ncta - 1) // ncta
    tpc = (rpc + 15) // 16
    R = (rpc + tpc - 1) // tpc
    return R, (N + R - 1) // R


def attn_items(nkeys):
    """(items, 32-key blocks per item) of a row of nkeys keys (sv_decode_flow.cu attn_split: <= 8 blocks per item)."""
    nblk = (nkeys + 31) // 32
    if nblk <= 8:
        return 1, nblk
    nact = min(MAXS, (nblk + 7) // 8)
    per = (nblk + nact - 1) // nact
    return (nblk + per - 1) // per, per


# ---- the decoder against hand-built buffers -------------------------------------------------------------------------------
def test_decode_rows_hand_built():
    B, n = 2, 24                                       # 3 fragments per row, rows 192 words apart
    words = np.zeros(B * 192, dtype=np.uint32)
    vals = torch.arange(B * n, dtype=torch.float32).view(B, n).bfloat16()
    bits = vals.view(torch.int16).numpy().astype(np.uint16).astype(np.uint32)
    for b in range(B):
        for i in range(n):
            words[b * 192 + (i // 8) * 64 + i % 8] = ((7 + b * 100 + i) << 16) | bits[b, i]
    words[5 * 8 + 3] = 0xFFFFFFFF                     # padding between fragments is never read
    got, tags = decode_rows(torch.from_numpy(words.view(np.int32)), B, n)
    assert torch.equal(got, vals) and got.is_contiguous()       # (the values go to the kernels as raw pointers)
    assert tags.tolist() == [[7 + b * 100 + i for i in range(n)] for b in range(B)]
    assert row_words(2048) == 256 * 64 and list(word_index(17)[[0, 7, 8, 9, 16]]) == [0, 7, 64, 65, 128]


def test_decode_partial_and_amax_hand_built():
    n_kv = 2
    words = np.zeros(2 * n_kv * MAXS * PSZ, dtype=np.uint64)
    b, h, c = 1, 1, 3
    base = ((b * n_kv + h) * MAXS + c) * PSZ
    m = np.arange(16, dtype=np.float32) - 3.5
    acc = np.linspace(-2, 2, 16 * D, dtype=np.float32)
    for k, v in enumerate(np.concatenate([m, m * 2, acc])):
        words[base + k] = (np.uint64(41 + k) << np.uint64(32)) | np.uint64(np.float32(v).view(np.uint32))
    (gm, gl, ga), tags = decode_partial(torch.from_numpy(words.view(np.int64)), b, h, c, n_kv)
    assert torch.equal(gm, torch.from_numpy(m)) and torch.equal(gl, torch.from_numpy(m * 2))
    assert torch.equal(ga, torch.from_numpy(acc).view(16, D)) and tags.tolist() == list(range(41, 41 + PSZ))
    amax = np.zeros(5 * 8, dtype=np.uint64)
    v = torch.tensor([1.5, -2.25]).bfloat16().view(torch.int16).numpy().astype(np.uint16)
    amax[3 * 8 + 0] = (np.uint64(0x1234) << np.uint64(48)) | (np.uint64(v[0]) << np.uint64(32)) | np.uint64(49156)
    amax[3 * 8 + 1] = (np.uint64(0x7FFF) << np.uint64(48)) | (np.uint64(v[1]) << np.uint64(32)) | np.uint64(7)
    t, val, idx = decode_amax(torch.from_numpy(amax.view(np.int64)), 5, 2)
    assert t[3].tolist() == [0x1234, 0x7FFF] and val[3].float().tolist() == [1.5, -2.25] and idx[3].tolist() == [49156, 7]


def test_tags_plans_and_item_split():
    assert tag16(0) == 1 and tag16(0x7FFF) == 0x8000 and tag16(0x8000) == 1 and tag32(0xFFFFFFFF) == 0
    assert plan(49156, 132) == (16, 3073) and plan(49157, 132) == (16, 3073) and plan(500, 132) == (4, 125)
    assert attn_items(256) == (1, 8) and attn_items(257) == (2, 5) and attn_items(8192) == (32, 8)
    assert attn_items(16384) == (64, 8) and attn_items(289) == (2, 5) and attn_items(1) == (1, 1)
