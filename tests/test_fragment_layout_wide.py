"""CPU replay of the index math of the 16-row ring GEMV phase (gemv_phase_wide in sv_decode_mega.cu, NG = 2).

One CTA tile of 16 weight rows over K = 2048 (two 1024-wide slabs, 8 consumer warps, 4 chunks of 32 per warp and slab) and
9-16 image rows in two groups of 8: group 0's activation fragments in registers, group 1's in the shared-memory block
(fragment i of consumer thread c at (i * NCT + c) * 16 bytes), each weight fragment feeding one m16n8k16 per group.  The
replay follows the kernel's expressions for the fragment loads, the LayerNorm statistics slots, the split-K reduction buffer
and the 16 x 16 epilogue (thread -> weight row n = tid & 15, image row mm = tid >> 4), the argmax partial index, and checks
the results against plain numpy, so an index error is caught without a GPU.
"""
import numpy as np
import pytest

from test_fragment_layout import mma_16816, words

NWC, CPW, NCT = 8, 4, 256
KS, NSTG = 1024, 2
K = KS * NSTG
CPS = KS // 32
CPWS = (CPS + NWC - 1) // NWC
MR = 16


def chunk(ks, warp, j):
    """(valid, first k) of chunk j of `warp` in slab ks (okc in the kernel)."""
    cl = warp + NWC * j
    return ks < NSTG and j < CPWS and cl < CPS, ks * KS + cl * 32


def group1_offset(i, tid):
    return (i * NCT + tid) * 16                     # xs + ((gi - 1) * 2 * CPW + i) * NCT * 16, gi = 1


def load_fragments(X, B):
    """reg[warp][lane][i] (group 0) and the shared-memory block (group 1), as the prologue fills them."""
    reg = np.zeros((NWC, 32, 2 * CPW, 8))
    smem = {}
    for warp in range(NWC):
        for lane in range(32):
            g, t, tid = lane >> 2, lane & 3, warp * 32 + lane
            for ks in range(2):
                for j in range(CPW):
                    ok, k0 = chunk(ks, warp, j)
                    i = ks * CPW + j
                    if ok and g < B:
                        reg[warp, lane, i] = X[g, k0 + 8 * t: k0 + 8 * t + 8]
                    off = group1_offset(i, tid)
                    assert off not in smem
                    smem[off] = X[g + 8, k0 + 8 * t: k0 + 8 * t + 8] if ok and g + 8 < B else np.zeros(8)
    return reg, smem


def test_group1_block_is_a_conflict_free_bijection():
    offs = sorted(group1_offset(i, tid) for i in range(2 * CPW) for tid in range(NCT))
    assert offs == list(range(0, 2 * CPW * NCT * 16, 16))          # X1_BYTES = 32 KB, every 16-byte slot once
    for i in range(2 * CPW):                                        # a warp's 128-bit loads: 32 consecutive 16-byte slots
        for warp in range(NWC):
            lanes = [group1_offset(i, warp * 32 + lane) for lane in range(32)]
            assert lanes == list(range(lanes[0], lanes[0] + 512, 16))


@pytest.mark.parametrize("B", [9, 12, 16])
def test_layernorm_statistics_slots(B):
    rng = np.random.default_rng(B)
    X = rng.standard_normal((16, K))
    reg, smem = load_fragments(X, B)
    stat = np.zeros(NWC * MR)
    for warp in range(NWC):
        for gi in range(2):
            for g in range(8):
                s = 0.0
                for t in range(4):                                   # quad_sum over the 4 lanes of row g
                    tid = warp * 32 + 4 * g + t
                    frags = reg[warp, 4 * g + t] if gi == 0 else [smem[group1_offset(i, tid)] for i in range(2 * CPW)]
                    s += float(np.sum(frags))
                stat[warp * MR + 8 * gi + g] = s
    for gi in range(2):
        for g in range(8):
            row = g + 8 * gi
            mean = sum(stat[w * MR + 8 * gi + g] for w in range(NWC)) / K
            np.testing.assert_allclose(mean, X[row].mean() if row < B else 0.0, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("B,R", [(16, 16), (9, 14), (13, 16)])
def test_two_group_tile_matches_matmul(B, R):
    rng = np.random.default_rng(100 + B)
    X = rng.standard_normal((16, K))
    X[B:] = rng.standard_normal((16 - B, K)) * 1e6                  # rows >= B must never reach the result
    W = rng.standard_normal((16, K))
    W[R:] = 0.0                                                      # rows past the tile are zero in the slot
    reg, smem = load_fragments(X, B)
    red = np.zeros(NWC * 16 * MR)
    for warp in range(NWC):
        c = [np.zeros((32, 4)), np.zeros((32, 4))]
        for ks in range(2):
            for j in range(CPW):
                ok, k0 = chunk(ks, warp, j)
                if not ok:
                    continue
                a1, a2 = [], []
                xv = [[], []]
                for lane in range(32):
                    g, t, tid = lane >> 2, lane & 3, warp * 32 + lane
                    lo = words(W[g, k0 + 8 * t: k0 + 8 * t + 8])               # lds16(sb + cl * 64)
                    hi = words(W[g + 8, k0 + 8 * t: k0 + 8 * t + 8])           # lds16(sb + 8 * pitch + cl * 64)
                    a1.append([lo[0], hi[0], lo[1], hi[1]])
                    a2.append([lo[2], hi[2], lo[3], hi[3]])
                    xv[0].append(words(reg[warp, lane, ks * CPW + j]))
                    xv[1].append(words(smem[group1_offset(ks * CPW + j, tid)]))
                for gi in range(2):
                    c[gi] = mma_16816(c[gi], a1, [[x[0], x[1]] for x in xv[gi]])
                    c[gi] = mma_16816(c[gi], a2, [[x[2], x[3]] for x in xv[gi]])
        for lane in range(32):
            g, t = lane >> 2, lane & 3
            for gi in range(2):
                red[(warp * 16 + g) * MR + 8 * gi + 2 * t] = c[gi][lane][0]
                red[(warp * 16 + g) * MR + 8 * gi + 2 * t + 1] = c[gi][lane][1]
                red[(warp * 16 + g + 8) * MR + 8 * gi + 2 * t] = c[gi][lane][2]
                red[(warp * 16 + g + 8) * MR + 8 * gi + 2 * t + 1] = c[gi][lane][3]
    Y = np.full((16, 16), np.nan)
    tile = 3
    amax = {}
    for tid in range(16 * MR):                                       # threadIdx.x < 16 * MR: one (n, mm) pair each
        n, mm = tid & 15, tid >> 4
        acc = sum(red[(w * 16 + n) * MR + mm] for w in range(NWC))
        if n < R and mm < B:
            Y[mm, n] = acc
        if n == 0 and mm < B:
            idx = tile * MR + mm
            assert idx not in amax
            amax[idx] = mm
    np.testing.assert_allclose(Y[:B, :R], X[:B] @ W[:R].T, rtol=1e-9, atol=1e-9)
    assert np.isnan(Y[B:]).all() and np.isnan(Y[:, R:]).all()
    assert sorted(amax) == list(range(tile * MR, tile * MR + B))    # partials [tile][16]: one slot per image row
