"""The decode-step kernels one launch at a time, against fp64 references (sv_op_attention_decode, sv_op_gemv_ring,
sv_op_rope_table, sv_op_rope).

Decode attention: the keys are built so that an error in the key range cannot hide in the tolerance.  Each query head is
aimed at up to three PROBE keys (the window start, keys 31/32/33, the first and last key of split / CTA ranges, the new
token at len - 1), each holding >= 20 % of its softmax mass, with distinctive V rows.  Every slot the kernel must not read
(len .. tcap - 1 and the keys below the window) holds a finite POISON key that would take > 99 % of the mass, with a large
V.  The output must be bitwise independent of the poison values.

Tolerances (calibrated on an H100 SXM 80 GB; the worst case of each kernel is printed as `CALIB` lines with -s):
  decode attention: |out - ref| <= 1 ulp(ref) + 0.02 rms(ref of that head)
  ring GEMV:        |y - ref| <= 1 ulp(ref) + 2^-18 sum_k |LN(x)_k w_nk| (+ 1 ulp of the pre-activation / pre-residual
                    value when there is one), and >= 99 % of the outputs bit-equal, on the kernel's own LayerNorm output;
                    that LayerNorm: within 1 ulp of fp64 (+ 2^-20 |mean| rstd |ln_w|) and >= 99.5 % bit-equal
  RoPE:             table within 1 bf16 ulp of transformers' Starcoder2RotaryEmbedding; rotation bit-exact
"""
import math

import pytest
import torch

from starvector_b200 import _lib
from starvector_b200 import engine as E

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 128
SPLIT, CLUSTER = _lib.SV_ATTN_DECODE_SPLIT, _lib.SV_ATTN_DECODE_CLUSTER
ATTN_ULPS, ATTN_C = 1.0, 0.02
PROBE_SCORE, POISON_SCORE = 11.0, 20.0      # q.k / sqrt(D) of a probe key / a poison key for every head of its group


def _ulp(x):
    """bf16 ulp of |x| (2^-133 floor for zeros)."""
    x = x.double().abs().clamp(min=2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(x)) - 7)


def _calib(name, ratio):
    print(f"CALIB {name}: worst error / tolerance = {ratio:.3f}")


# ---- decode attention --------------------------------------------------------------------------------------------------
def _key_lo(n, window):
    return max(0, n - window) if window > 0 else 0


def _ranges(n, window, parts):
    """(first, last) key of every split / CTA that gets keys, by the kernels' `per` rule over 32-key blocks."""
    lo = _key_lo(n, window)
    blk_lo, blk_hi = lo // 32, (n + 31) // 32
    per = (blk_hi - blk_lo + parts - 1) // parts
    out = []
    for s in range(parts):
        b0 = blk_lo + s * per
        b1 = min(blk_hi, b0 + per)
        if b0 < b1:
            out.append((max(lo, b0 * 32), min(n, b1 * 32) - 1))
    return out


def _nsplit_for(n):        # sv_engine.cu nsplit_for
    return max(1, min(128, (n + 31) // 32))


def _ncta_for(n):          # attention_decode_cluster_ncta
    return max(1, min(8, ((n + 31) // 32 + 7) // 8))


class AttnCase:
    """B rows of qkv plus their caches (tcap slots), probes and poison; `ref` is the fp64 attention rounded to bf16."""

    def __init__(self, B, nh, nkv, lens, tcap, window, parts, seed):
        self.B, self.nh, self.nkv, self.lens, self.tcap, self.window = B, nh, nkv, list(lens), tcap, window
        g = torch.Generator(device=DEV).manual_seed(seed)
        grp = nh // nkv
        f64 = dict(device=DEV, dtype=torch.float64)
        # orthonormal query directions inside each group: a key along u_h scores only for head h
        u = torch.linalg.qr(torch.randn(B * nkv, D, grp, generator=g, **f64)).Q.transpose(1, 2).reshape(B, nkv, grp, D)
        q = u * math.sqrt(D)                                            # a N(0,1) key scores N(0,1)
        K = torch.randn(B, nkv, tcap, D, generator=g, **f64)
        V = torch.randn(B, nkv, tcap, D, generator=g, **f64)
        self.probes = {}
        for b, n in enumerate(self.lens):
            lo = _key_lo(n, window)
            cand = [n - 1, lo, 31, 32, 33]
            for p in parts:
                for a, z in _ranges(n, window, p):
                    cand += [a, z]
            seen, uniq = set(), []
            for c in cand:
                if lo <= c < n and c not in seen:
                    seen.add(c)
                    uniq.append(c)
            for kvh in range(nkv):
                for i, pos in enumerate(uniq[:3 * grp]):
                    h = (i + kvh) % grp
                    K[b, kvh, pos] = u[b, kvh, h] * PROBE_SCORE
                    V[b, kvh, pos] = 4.0 * torch.randn(D, generator=g, **f64)
                    self.probes.setdefault((b, kvh * grp + h), []).append(pos)
        self.q = q.reshape(B, nh, D).to(torch.bfloat16)
        self.K, self.V = K.to(torch.bfloat16), V.to(torch.bfloat16)
        self.u = u
        self.qkv = torch.randn(B, (nh + 2 * nkv) * D, generator=g, device=DEV).to(torch.bfloat16)
        self.qkv[:, :nh * D] = self.q.reshape(B, nh * D)
        self.ref, self.rms = self._reference()
        self.kc, self.vc = self._caches(POISON_SCORE, 500.0)

    def _caches(self, score, vpoison):
        """kcache / vtcache with every slot outside each row's key range poisoned."""
        K, V = self.K.clone(), self.V.clone()
        poison = (self.u.sum(2) * score).to(torch.bfloat16)               # [B, nkv, D]: scores `score` for every head
        for b, n in enumerate(self.lens):
            lo = _key_lo(n, self.window)
            for sl in (slice(0, lo), slice(n, self.tcap)):
                K[b, :, sl] = poison[b, :, None]
                V[b, :, sl] = vpoison
        return K.contiguous(), V.transpose(2, 3).contiguous()

    def _reference(self):
        grp = self.nh // self.nkv
        ref = torch.empty(self.B, self.nh, D, device=DEV, dtype=torch.float64)
        q, K, V = self.q.double(), self.K.double(), self.V.double()
        for b, n in enumerate(self.lens):
            lo = _key_lo(n, self.window)
            for kvh in range(self.nkv):
                hs = slice(kvh * grp, (kvh + 1) * grp)
                p = torch.softmax(q[b, hs] @ K[b, kvh, lo:n].T / math.sqrt(D), dim=-1)
                ref[b, hs] = p @ V[b, kvh, lo:n]
                for h in range(grp):           # the construction's promise: every probe holds >= 20 % of its head's mass
                    for pos in self.probes.get((b, kvh * grp + h), []):
                        assert p[h, pos - lo] >= 0.2, (b, kvh, h, pos, float(p[h, pos - lo]))
        rms = ref.pow(2).mean(-1, keepdim=True).sqrt()
        return ref, rms

    def run(self, impl, parts, per_row, kc=None, vc=None):
        kc = self.kc if kc is None else kc
        vc = self.vc if vc is None else vc
        return E.op_attention_decode(self.qkv, kc, vc, self.lens, self.nh, self.nkv, parts, self.window, impl, per_row)

    def tol(self):
        return ATTN_ULPS * _ulp(self.ref) + ATTN_C * self.rms

    def check(self, impl, parts, per_row):
        """Returns the output after the value, determinism and poison checks; the worst error / tolerance in self.worst."""
        out = self.run(impl, parts, per_row)
        assert bool(torch.isfinite(out.float()).all())
        o = out.view(self.B, self.nh, D).double()
        ratio = ((o - self.ref).abs() / self.tol()).max().item()
        self.worst = max(getattr(self, "worst", 0.0), ratio)
        if ratio > 1:
            bad = ((o - self.ref).abs() > self.tol()).nonzero()[:5].tolist()
            raise AssertionError(f"impl {impl} parts {parts} per_row {per_row} lens {self.lens}: worst err/tol {ratio:.2f} "
                                 f"at (row, head, dim) {bad}")
        assert torch.equal(out, self.run(impl, parts, per_row)), "repeated launches differ"
        kc2, vc2 = self._caches(POISON_SCORE - 3.0, -300.0)
        assert torch.equal(out, self.run(impl, parts, per_row, kc2, vc2)), "the output depends on excluded slots"
        return out


TCAP = 4384
LENGTHS = [1, 2, 31, 32, 33, 64, 65, 257, 2047, 2048, 2049, 4355, TCAP - 1]


def _parts(impl, n):
    if impl == SPLIT:   # the per-op rule at this length, generate's rule (fixed from prefix + max_new), 1, 7 and 128
        return sorted({1, 7, 128, _nsplit_for(n), _nsplit_for(min(TCAP, n + 2000))})
    return sorted({1, 3, 8, _ncta_for(n), _ncta_for(min(TCAP, n + 2000))})


@pytest.mark.parametrize("per_row", [0, 1], ids=["plain", "rows"])
@pytest.mark.parametrize("impl", [SPLIT, CLUSTER], ids=["split", "cluster"])
@pytest.mark.parametrize("n", LENGTHS)
def test_decode_attention_lengths(n, impl, per_row):
    """Every split / CTA count the engine can pick at this length, including 8-CTA clusters whose CTAs mostly get no keys."""
    lens = [n, n] if not per_row else [n, max(1, n // 3)]
    parts = _parts(impl, n)
    c = AttnCase(2, 16, 1, lens, TCAP, 0, parts, seed=n * 4 + impl * 2 + per_row)
    other = CLUSTER if impl == SPLIT else SPLIT
    for p in parts:
        out = c.check(impl, p, per_row)
        # split and cluster agree within the tolerance
        alt = c.run(other, min(p, 8) if other == CLUSTER else p, per_row)
        assert bool(((out.view_as(c.ref).double() - alt.view_as(c.ref).double()).abs() <= c.tol()).all())
        if per_row:   # the session kernels are the plain kernels, row by row, at the same length and split count
            for b, nb in enumerate(lens):
                one = E.op_attention_decode(c.qkv[b:b + 1], c.kc[b:b + 1], c.vc[b:b + 1], [nb], 16, 1, p, 0, impl, False)
                assert torch.equal(one[0], out[b]), (b, nb, p)
    _calib(f"attention_decode impl={impl} n={n} per_row={per_row}", c.worst)


WINDOW_CASES = [(0, [300, 300]), (24, [23, 24, 25]), (4096, [4095, 4096, 4097]), (100, [99, 100, 101])]


@pytest.mark.parametrize("impl", [SPLIT, CLUSTER], ids=["split", "cluster"])
@pytest.mark.parametrize("window,lens", WINDOW_CASES, ids=["w0", "w24", "w4096", "w100"])
@pytest.mark.parametrize("nh,nkv", [(16, 1), (36, 4), (4, 2), (2, 1)])
def test_decode_attention_groups_and_windows(nh, nkv, window, lens, impl):
    """Sliding windows at lengths window - 1, window and window + 1 (the session kernels, rows of different lengths)."""
    tcap = 4128 if window >= 4096 else 320
    parts = [1, 5, 8] if impl == CLUSTER else [1, 5, 64, _nsplit_for(max(lens))]
    c = AttnCase(len(lens), nh, nkv, lens, tcap, window, parts, seed=window + nh * 7 + impl)
    for p in parts:
        out = c.check(impl, p, 1)
        for b, nb in enumerate(lens):
            one = E.op_attention_decode(c.qkv[b:b + 1], c.kc[b:b + 1], c.vc[b:b + 1], [nb], nh, nkv, p, window, impl, False)
            assert torch.equal(one[0], out[b]), (b, nb, p)
    _calib(f"attention_decode impl={impl} group={nh}/{nkv} window={window}", c.worst)


@pytest.mark.parametrize("impl", [SPLIT, CLUSTER], ids=["split", "cluster"])
@pytest.mark.parametrize("B", [1, 8, 9, 16])
def test_decode_attention_batches(B, impl):
    """Session rows of very different lengths side by side (1 next to 4000), 36 heads over 4 KV heads."""
    g = torch.Generator().manual_seed(B)
    lens = [1, 4000, 33, 2049] + torch.randint(1, 4001, (12,), generator=g).tolist()
    lens = lens[:B]
    top = max(lens)
    parts = [_ncta_for(top), 8] if impl == CLUSTER else [_nsplit_for(top), 128]
    c = AttnCase(B, 36, 4, lens, 4096, 0, parts, seed=100 + B + impl)
    for p in parts:
        out = c.check(impl, p, 1)
        for b, nb in enumerate(lens):
            one = E.op_attention_decode(c.qkv[b:b + 1], c.kc[b:b + 1], c.vc[b:b + 1], [nb], 36, 4, p, 0, impl, False)
            assert torch.equal(one[0], out[b]), (b, nb, p)
    _calib(f"attention_decode impl={impl} B={B}", c.worst)


class MapAttnCase:
    """The column map of a speculative verify step: ncols query columns over ONE cache row holding L0 prefix keys plus the
    live columns' own keys; column c attends to keys [0, pos[c]].  The slot of each column and the slot right after it
    (pos[c] + 1, the next column's key) hold a probe aimed at one head of that column (score ~11 against N(0, 1) for the
    other keys), so a column that reads one key too many or too few is far outside the tolerance.  Cache rows 1..15, which
    no column may read, hold other keys."""

    ROWS = 16

    def __init__(self, nh, nkv, ncols, n_live, L0, tcap, seed):
        self.nh, self.nkv, self.ncols, self.tcap = nh, nkv, ncols, tcap
        self.pos = _map_positions(ncols, n_live, L0)
        g = torch.Generator(device=DEV).manual_seed(seed)
        grp = nh // nkv
        f64 = dict(device=DEV, dtype=torch.float64)
        q = torch.randn(ncols, nkv, grp, D, generator=g, **f64)
        u = q / q.norm(dim=-1, keepdim=True)                            # column c, head h's direction
        K = torch.randn(self.ROWS, nkv, tcap, D, generator=g, **f64)
        V = torch.randn(self.ROWS, nkv, tcap, D, generator=g, **f64)
        aimed = {}                                                      # (kv head, slot) -> the directions aimed at it
        for c, p in enumerate(self.pos):
            for kvh in range(nkv):
                for slot in (p, p + 1):
                    if slot < tcap:
                        aimed.setdefault((kvh, slot), []).append(u[c, kvh, (c + kvh) % grp])
        for (kvh, slot), dirs in aimed.items():
            K[0, kvh, slot] = sum(dirs) * PROBE_SCORE
            V[0, kvh, slot] = 4.0 * torch.randn(D, generator=g, **f64)
        self.q = (u * math.sqrt(D)).reshape(ncols, nh, D).to(torch.bfloat16)
        self.qkv = torch.randn(ncols, (nh + 2 * nkv) * D, generator=g, device=DEV).to(torch.bfloat16)
        self.qkv[:, :nh * D] = self.q.reshape(ncols, nh * D)
        Kb, Vb = K.to(torch.bfloat16), V.to(torch.bfloat16)
        self.kc, self.vc = Kb.contiguous(), Vb.transpose(2, 3).contiguous()
        qd, Kd, Vd = self.q.double(), Kb.double(), Vb.double()
        self.ref = torch.empty(ncols, nh, D, **f64)
        for c, p in enumerate(self.pos):
            for kvh in range(nkv):
                hs = slice(kvh * grp, (kvh + 1) * grp)
                w = torch.softmax(qd[c, hs] @ Kd[0, kvh, :p + 1].T / math.sqrt(D), dim=-1)
                self.ref[c, hs] = w @ Vd[0, kvh, :p + 1]
        self.rms = self.ref.pow(2).mean(-1, keepdim=True).sqrt()

    def run(self, ncta, kc=None, vc=None):
        return E.op_attention_decode(self.qkv, self.kc if kc is None else kc, self.vc if vc is None else vc, self.pos, self.nh,
                                     self.nkv, ncta, 0, CLUSTER, 2)

    def poisoned(self, after):
        """Caches whose row-0 slots > after and whose other rows hold other finite values."""
        kc, vc = self.kc.clone(), self.vc.clone()
        kc[0, :, after + 1:] = 2.0
        vc[0, :, :, after + 1:] = 300.0
        kc[1:] = -3.0 * kc[1:]
        vc[1:] = 500.0
        return kc, vc


def _map_l0s(ncta, tcap):
    """31/32/33, the first and last key of each CTA's 32-key block range at ~1100 keys with this cluster size, tcap - 16."""
    edges = {31, 32, 33, tcap - 16}
    for a, z in _ranges(1100, 0, ncta)[:3]:
        edges.update({a, z, z + 1})
    return sorted(edges)


@pytest.mark.parametrize("ncta", [1, 2, 3, 4, 5, 6, 7, 8])
def test_decode_attention_column_map(ncta):
    """attention_decode_cluster_map_kernel against fp64, and bitwise against the plain cluster kernel at each column's
    length with the same cluster size (the verify step's bit-identity with plain decoding).  Columns at L0 + c, inert ones
    at the last live position; 8-CTA clusters over short rows (the engine sizes the cluster from prefix + max_new)."""
    tcap = 2080
    worst = 0.0
    cases = [(16, 1, 16, 16), (4, 2, 9, 5)]
    for i, L0 in enumerate(_map_l0s(ncta, tcap)):
        nh, nkv, ncols, n_live = cases[i % len(cases)]
        if i % 3 == 2:
            n_live = 1
        c = MapAttnCase(nh, nkv, ncols, n_live, L0, tcap, seed=ncta * 1000 + L0)
        out = c.run(ncta)
        assert bool(torch.isfinite(out.float()).all())
        o = out.view(ncols, nh, D).double()
        tol = ATTN_ULPS * _ulp(c.ref) + ATTN_C * c.rms
        ratio = ((o - c.ref).abs() / tol).max().item()
        worst = max(worst, ratio)
        assert ratio <= 1.0, (L0, ncols, n_live, ratio, ((o - c.ref).abs() > tol).nonzero()[:5].tolist())
        assert torch.equal(out, c.run(ncta)), "repeated launches differ"
        for col, p in enumerate(c.pos):
            one = E.op_attention_decode(c.qkv[col:col + 1], c.kc[:1], c.vc[:1], [p + 1], nh, nkv, ncta, 0, CLUSTER, 0)
            assert torch.equal(one[0], out[col]), (L0, col, p)
        for p in sorted(set(c.pos)):
            kc, vc = c.poisoned(p)
            alt = c.run(ncta, kc, vc)
            for col, pc in enumerate(c.pos):
                if pc <= p:
                    assert torch.equal(alt[col], out[col]), f"column {col} (pos {pc}) reads a slot > {p} or another row"
    _calib(f"attention_decode column map ncta={ncta}", worst)


# ---- RoPE ----------------------------------------------------------------------------------------------------------------
def _hf_rope_table(theta, max_pos, d=128):
    """cos / sin [max_pos, d / 2] as transformers' Starcoder2RotaryEmbedding returns them in bf16, with the oracle's config."""
    from transformers import Starcoder2Config
    from transformers.models.starcoder2.modeling_starcoder2 import Starcoder2RotaryEmbedding

    cfg = Starcoder2Config(hidden_size=d * 4, num_attention_heads=4, num_key_value_heads=2, max_position_embeddings=max_pos,
                           rope_parameters={"rope_type": "default", "rope_theta": float(theta)})
    rot = Starcoder2RotaryEmbedding(config=cfg)
    cos, sin = rot(torch.zeros(1, dtype=torch.bfloat16), torch.arange(max_pos)[None])
    return cos[0, :, : d // 2], sin[0, :, : d // 2]


@pytest.mark.parametrize("theta", [1e4, 1e6])
def test_rope_table_matches_transformers(theta):
    max_pos = 16384
    cos, sin = E.op_rope_table(max_pos, D, theta)
    hc, hs = _hf_rope_table(theta, max_pos)
    for name, got, ref in (("cos", cos.cpu(), hc), ("sin", sin.cpu(), hs)):
        err = (got.double() - ref.double()).abs()
        ratio = (err / _ulp(ref)).max().item()
        diff = (err > 0).double().mean().item()
        print(f"CALIB rope_table theta={theta:g} {name}: {100 * diff:.4f} % of entries differ, worst {ratio:.2f} ulp")
        assert ratio <= 1.0, f"{name}: {ratio:.2f} ulp at {int(err.argmax()) // (D // 2)}"


def _rope_ref(x, pos, cos_t, sin_t):
    """transformers' apply_rotary_pos_emb on bf16 tensors: x [rows, heads, D] at positions pos [rows] (three bf16 ops)."""
    c = torch.cat([cos_t, cos_t], -1)[pos][:, None]
    s = torch.cat([sin_t, sin_t], -1)[pos][:, None]
    rot = torch.cat([-x[..., D // 2:], x[..., : D // 2]], -1)
    return (x * c) + (rot * s)


def _rope_setup(rows, nh, nkv, max_pos, seed):
    g = torch.Generator().manual_seed(seed)
    cos, sin = E.op_rope_table(max_pos, D, 1e4)
    qkv = torch.randn(rows, (nh + 2 * nkv) * D, generator=g).to(torch.bfloat16)
    return qkv, cos.cpu(), sin.cpu()


@pytest.mark.parametrize("pos0,seq,rows", [(0, 5, 10), (37, 5, 10), (60, 8, 8), (0, 1, 3)])
def test_rope_prefill_bit_exact(pos0, seq, rows):
    """Row r at pos0 + r % seq; positions past the 64-entry table use its last entry (pos0 = 60)."""
    nh, nkv, max_pos = 4, 2, 64
    qkv, cos, sin = _rope_setup(rows, nh, nkv, max_pos, seed=pos0 + seq)
    got = E.op_rope(qkv.cuda(), cos.cuda(), sin.cuda(), nh, nkv, seq=seq, pos0=pos0).cpu()
    pos = (pos0 + torch.arange(rows) % seq).clamp(max=max_pos - 1)
    x = qkv.view(rows, nh + 2 * nkv, D)
    ref = x.clone()
    ref[:, : nh + nkv] = _rope_ref(x[:, : nh + nkv], pos, cos, sin)
    assert torch.equal(got.view_as(ref), ref)


@pytest.mark.parametrize("per_row", [0, 1], ids=["plain", "rows"])
@pytest.mark.parametrize("append", [False, True], ids=["rope", "rope_append"])
def test_rope_decode_bit_exact(append, per_row):
    """One token per row: q (and k) rotated; with the append kernel, rotated k and v land in the caches at the row's position,
    nothing else changes, and a row at pos >= tcap writes nothing.  Positions past the table use its last entry."""
    nh, nkv, max_pos, tcap = 4, 2, 64, 96
    pos = [5, 70, 0, 96, 63, 95] if per_row else [70] * 6
    rows = len(pos)
    qkv, cos, sin = _rope_setup(rows, nh, nkv, max_pos, seed=3 + per_row)
    g = torch.Generator().manual_seed(9)
    kc = torch.randn(rows, nkv, tcap, D, generator=g).to(torch.bfloat16)
    vc = torch.randn(rows, nkv, D, tcap, generator=g).to(torch.bfloat16)
    kd, vd = kc.cuda(), vc.cuda()
    got = E.op_rope(qkv.cuda(), cos.cuda(), sin.cuda(), nh, nkv, pos=pos, per_row=bool(per_row),
                    kcache=kd if append else None, vtcache=vd if append else None).cpu()
    x = qkv.view(rows, nh + 2 * nkv, D)
    tp = torch.tensor(pos).clamp(max=max_pos - 1)
    rot = _rope_ref(x[:, : nh + nkv], tp, cos, sin)
    ref = x.clone()
    if append:
        ref[:, :nh] = rot[:, :nh]
        assert torch.equal(got.view_as(ref), ref)              # k and v columns of qkv are left as they were
        kref, vref = kc.clone(), vc.clone()
        for b, p in enumerate(pos):
            if p < tcap:
                kref[b, :, p] = rot[b, nh:]
                vref[b, :, :, p] = x[b, nh + nkv:]
        assert torch.equal(kd.cpu(), kref) and torch.equal(vd.cpu(), vref)
    else:
        ref[:, : nh + nkv] = rot
        assert torch.equal(got.view_as(ref), ref)


# ---- weight-ring GEMV ----------------------------------------------------------------------------------------------------
def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ragged_n():
    """An N whose tiles have R < 16 rows and a ragged last tile with one CTA per SM (2113 on a 132-SM part)."""
    nsm = _nsm()
    n = 16 * nsm + 1
    while True:
        rpc = (n + nsm - 1) // nsm
        tpc = (rpc + 15) // 16
        r = (rpc + tpc - 1) // tpc
        if r < 16 and n % r:
            return n
        n += 1


def _ln_rows(B, K, g):
    """x rows: N(0,1); every third row has a large mean (30 + N(0,1)); the last row of >= 3 is constant."""
    x = torch.randn(B, K, generator=g, device=DEV, dtype=torch.float64)
    x[1::3] += 30.0
    if B >= 3:
        x[-1] = 3.0
    return x.to(torch.bfloat16)


def _ln_ref(x, ln, eps=1e-5):
    xd = x.double()
    mu = xd.mean(-1, keepdim=True)
    var = (xd - mu).pow(2).mean(-1, keepdim=True)
    return ((xd - mu) / torch.sqrt(var + eps) * ln[0].double() + ln[1].double()).to(torch.bfloat16)


def _kernel_ln(x, ln, eps=1e-5):
    """The ring kernel's own bf16 LayerNorm output: the same launch over an identity weight (every dot product is one exact
    product, so y = LN(x) as the kernel rounded it)."""
    K = x.shape[1]
    eye = torch.eye(K, device=DEV, dtype=torch.bfloat16)
    return E.op_gemv_ring(x, eye, None, None, ln, ln_eps=eps)


def _ring_ref(x, w, bias=None, res=None, ln=None, act=0, eps=1e-5):
    """fp64 with the kernel's rounding points: dot, + bias -> bf16, act -> bf16, + residual -> bf16, on the kernel's own
    LayerNorm output (checked against fp64 on its own in test_gemv_ring_layernorm: a 1-ulp LayerNorm difference in one
    column moves every output of the row).  Returns (reference, absolute floor of the tolerance, the GEMV input)."""
    xd = x.double() if ln is None else _kernel_ln(x, ln, eps).double()
    wd = w.double()
    acc = xd @ wd.T
    y = acc + (bias.double() if bias is not None else 0.0)
    y = y.to(torch.bfloat16).double()
    # absolute floor: fp32 accumulation over K, and a 1-ulp difference at the first rounding point carried through the
    # activation / residual rounding points (where the final value can be much smaller than the pre-residual one)
    scale = 2.0 ** -18 * (xd.abs() @ wd.abs().T) + (_ulp(y) if act or res is not None else 0.0)
    if act == _lib.SV_ACT_GELU_TANH:
        y = torch.nn.functional.gelu(y, approximate="tanh").to(torch.bfloat16).double()
    elif act != 0:
        raise ValueError(act)
    if res is not None:
        y = (y + res.double()).to(torch.bfloat16).double()
    return y, scale, xd


def _ring_check(y, ref, floor, name):
    y = y.double()
    tol = _ulp(ref) + floor
    err = (y - ref).abs()
    ratio = (err / tol).max().item()
    eq = (y == ref).double().mean().item()
    print(f"CALIB gemv_ring {name}: worst error / tolerance = {ratio:.3f}, bit-equal {100 * eq:.3f} %")
    assert ratio <= 1.0, f"{name}: worst err/tol {ratio:.2f} at {divmod(int((err / tol).argmax()), y.shape[1])}"
    assert eq >= 0.99, f"{name}: only {100 * eq:.2f} % bit-equal"


def _weights(N, K, g, bias=True):
    w = (torch.randn(N, K, generator=g, device=DEV) / math.sqrt(K)).to(torch.bfloat16)
    b = (torch.randn(N, generator=g, device=DEV) * 0.1).to(torch.bfloat16) if bias else None
    return w, b


def _ln_params(K, g):
    return ((1.0 + 0.3 * torch.randn(K, generator=g, device=DEV)).to(torch.bfloat16),
            (0.2 * torch.randn(K, generator=g, device=DEV)).to(torch.bfloat16))


# (name, N, K, LayerNorm, act, residual, max rows)
RING_SHAPES = [
    ("v1 c_attn 2304x2048 LN", 2304, 2048, True, 0, False, 16),
    ("v1 c_proj 2048x2048 +res in place", 2048, 2048, False, 0, True, 16),
    ("v1 c_fc 8192x2048 LN gelu", 8192, 2048, True, _lib.SV_ACT_GELU_TANH, False, 16),
    ("v1 c_fc2 2048x8192 +res", 2048, 8192, False, 0, True, 16),
    ("v2 c_attn 5632x4608 LN", 5632, 4608, True, 0, False, 8),
    ("v2 mlp_c_proj 4608x18432 +res", 4608, 18432, False, 0, True, 16),
    ("K96 LN", "ragged", 96, True, 0, False, 8),
    ("K640 LN gelu", "ragged", 640, True, _lib.SV_ACT_GELU_TANH, False, 8),
    ("K1024 LN", "ragged", 1024, True, 0, True, 16),
    ("K1536 LN", "ragged", 1536, True, 0, False, 16),
    ("K640 plain", "ragged", 640, False, 0, True, 16),
]


@pytest.mark.parametrize("name,N,K,has_ln,act,has_res,max_rows", RING_SHAPES, ids=[s[0] for s in RING_SHAPES])
def test_gemv_ring_shapes(name, N, K, has_ln, act, has_res, max_rows):
    """Every row count in {1, 3, 8, 9, 13, 16} the shape has kernels for; the slab-tiled path is bitwise the plain one,
    16 rows are bitwise two launches of 8."""
    N = _ragged_n() if N == "ragged" else N
    g = torch.Generator(device=DEV).manual_seed(N + K)
    w, b = _weights(N, K, g)
    ln = _ln_params(K, g) if has_ln else None
    x16 = _ln_rows(16, K, g)
    r16 = torch.randn(16, N, generator=g, device=DEV).to(torch.bfloat16) if has_res else None
    for B in [1, 3, 8, 9, 13, 16]:
        if B > max_rows:
            continue
        x, res = x16[:B].contiguous(), (r16[:B].clone() if has_res else None)
        ref, scale, _ = _ring_ref(x, w, b, res, ln, act)
        if has_res:      # in place, as the engine runs it: y aliases the residual
            y = res.clone()
            E.op_gemv_ring(x, w, b, y, ln, act, y=y)
        else:
            y = E.op_gemv_ring(x, w, b, None, ln, act)
        _ring_check(y, ref, scale, f"{name} B={B}")
        yt = E.op_gemv_ring(x, w, b, res, ln, act, tiled=True)
        assert torch.equal(yt, y), "slab-tiled copy differs from the row-major stream"
        if B == 16:
            lo = E.op_gemv_ring(x[:8].contiguous(), w, b, res[:8].contiguous() if has_res else None, ln, act)
            hi = E.op_gemv_ring(x[8:].contiguous(), w, b, res[8:].contiguous() if has_res else None, ln, act)
            assert torch.equal(torch.cat([lo, hi]), y), "16 rows differ from two launches of 8"


@pytest.mark.parametrize("K", [96, 640, 1024, 1536, 2048, 4608])
def test_gemv_ring_layernorm(K):
    """The fused LayerNorm, register-resident (two slabs or fewer) and streamed (more, e.g. K = 96 and 640, 32- and 128-wide
    slabs; and v2's 4608): within 1 bf16 ulp of fp64 (plus the fp32 cancellation floor of large-mean rows) everywhere and
    bit-equal for >= 99.5 %, rows with a mean of 30 + N(0,1) included; a constant row gives exactly ln_b."""
    g = torch.Generator(device=DEV).manual_seed(K)
    ln = _ln_params(K, g)
    for B in ([1, 8] if K in (96, 640, 4608) else [1, 9, 16]):
        x = _ln_rows(B, K, g)
        got = _kernel_ln(x, ln).double()
        ref = _ln_ref(x, ln).double()
        # fp32 statistics: x - mean cancels on rows with a large mean, leaving the mean's fp32 error (~2^-20 |mean|, times
        # rstd and the affine weight) on outputs near zero
        xd = x.double()
        floor = 2.0 ** -20 * xd.mean(-1, keepdim=True).abs() / (xd.var(-1, unbiased=False, keepdim=True) + 1e-5).sqrt()
        err = (got - ref).abs() / (_ulp(ref) + floor * ln[0].double().abs())
        eq = (got == ref).double().mean().item()
        print(f"CALIB gemv_ring LayerNorm K={K} B={B}: worst {err.max().item():.2f} ulp, bit-equal {100 * eq:.3f} %")
        assert err.max().item() <= 1.0 and eq >= 0.995
        if B >= 3:
            assert torch.equal(got[-1], ln[1].double())


def test_gemv_ring_matches_linear_rowgroup():
    g = torch.Generator(device=DEV).manual_seed(5)
    for B, N, K in [(3, 2304, 2048), (16, 2048, 8192)]:
        w, b = _weights(N, K, g)
        x = torch.randn(B, K, generator=g, device=DEV).to(torch.bfloat16)
        y = E.op_gemv_ring(x, w, b).double()
        lin = E.op_linear(x, w, b, None, 0, _lib.SV_LINEAR_ROWGROUP).double()
        _, floor, _ = _ring_ref(x, w, b)
        assert bool(((y - lin).abs() <= _ulp(lin) + floor).all())
        assert (y == lin).double().mean().item() >= 0.99


def test_gemv_ring_constant_row_gives_ln_bias():
    """A constant row normalises to exactly ln_b: the GEMV then sees ln_b itself."""
    g = torch.Generator(device=DEV).manual_seed(6)
    K, N = 2048, 2304
    w, b = _weights(N, K, g)
    ln = _ln_params(K, g)
    x = torch.full((2, K), 3.0, device=DEV).to(torch.bfloat16)
    y = E.op_gemv_ring(x, w, b, None, ln)
    plain = E.op_gemv_ring(torch.stack([ln[1], ln[1]]), w, b)          # the same GEMV on ln_b, without the LayerNorm
    assert torch.equal(y, plain)


def _map_positions(ncols, n_live, cur):
    """svspec::set_map: live column c at cur + c, inert columns at the last live position (cur - 1 when n_live = 0)."""
    return [cur + c if c < n_live else cur + n_live - 1 for c in range(ncols)]


@pytest.mark.parametrize("per_row", [0, 1, 2], ids=["plain", "rows", "map"])
@pytest.mark.parametrize("B", [1, 2, 3, 8, 9, 13, 16])
@pytest.mark.parametrize("nh,nkv", [(16, 1), (4, 2)])
def test_gemv_ring_qkv_appends_kv(nh, nkv, B, per_row):
    """The QKV epilogue changes the caches only at (row, kv head, pos), with y's K / V columns; pos == tcap writes nothing.
    The column map of a verify step (per_row = 2, B columns of cache row 0): live columns append at their positions, which
    straddle a 32-slot edge or end at tcap - 1; inert columns write nothing, not even at the last live position they point
    to (cur - 1 with no live column, a slot holding data); y is bitwise the plain QKV launch's; the other cache rows keep
    every byte.  Row-major and slab-tiled weights."""
    K, tcap = 2048, 128
    N = (nh + 2 * nkv) * D
    g = torch.Generator(device=DEV).manual_seed(B * 10 + per_row)
    w, b = _weights(N, K, g)
    ln = _ln_params(K, g)
    x = _ln_rows(B, K, g)
    ref, scale, _ = _ring_ref(x, w, b, None, ln)
    if per_row == 2:
        bf = dict(dtype=torch.bfloat16, device=DEV)
        for n_live in sorted({0, 1, B - 1, B}):
            for cur in (96 - n_live // 2, tcap - n_live) if n_live else (96, tcap):
                pos = _map_positions(B, n_live, cur)
                for tiled in (False, True):
                    kc = torch.randn(3, nkv, tcap, D, generator=g, device=DEV).to(torch.bfloat16)
                    vc = torch.randn(3, nkv, D, tcap, generator=g, device=DEV).to(torch.bfloat16)
                    k0, v0 = kc.clone(), vc.clone()
                    y = E.op_gemv_ring(x, w, b, None, ln, epi=1, kcache=kc, vtcache=vc, n_head=nh, n_kv=nkv, pos=pos,
                                       per_row=2, n_live=n_live, tiled=tiled)
                    # the plain launch on the same inputs (B cache rows, as it reads them; pos = tcap: it writes nothing)
                    plain = E.op_gemv_ring(x, w, b, None, ln, epi=1, kcache=torch.zeros(B, nkv, tcap, D, **bf),
                                           vtcache=torch.zeros(B, nkv, D, tcap, **bf), n_head=nh, n_kv=nkv, pos=[tcap],
                                           tiled=tiled)
                    assert torch.equal(y, plain), (n_live, cur, tiled)
                    kexp, vexp = k0.clone(), v0.clone()
                    ky = y[:, nh * D:(nh + nkv) * D].view(B, nkv, D)
                    vy = y[:, (nh + nkv) * D:].view(B, nkv, D)
                    for c in range(n_live):
                        kexp[0, :, pos[c]] = ky[c]
                        vexp[0, :, :, pos[c]] = vy[c]
                    assert torch.equal(kc, kexp) and torch.equal(vc, vexp), (n_live, cur, tiled)
        _ring_check(y, ref, scale, f"qkv {nh}/{nkv} B={B} per_row=map")
        return
    pos_sets = [[(7 * r + 3) % tcap for r in range(B)], [tcap] * B] if per_row else [[77] * B, [tcap] * B]
    if per_row and B > 1:
        pos_sets[0][1] = tcap                       # one row past the cache: nothing written for it
    for pos in pos_sets:
        kc = torch.randn(B, nkv, tcap, D, generator=g, device=DEV).to(torch.bfloat16)
        vc = torch.randn(B, nkv, D, tcap, generator=g, device=DEV).to(torch.bfloat16)
        k0, v0 = kc.clone(), vc.clone()
        y = E.op_gemv_ring(x, w, b, None, ln, epi=1, kcache=kc, vtcache=vc, n_head=nh, n_kv=nkv, pos=pos,
                           per_row=bool(per_row))
        _ring_check(y, ref, scale, f"qkv {nh}/{nkv} B={B} per_row={per_row}")
        kexp, vexp = k0.clone(), v0.clone()
        ky = y[:, nh * D:(nh + nkv) * D].view(B, nkv, D)
        vy = y[:, (nh + nkv) * D:].view(B, nkv, D)
        for r in range(B):
            if pos[r] < tcap:
                kexp[r, :, pos[r]] = ky[r]
                vexp[r, :, :, pos[r]] = vy[r]
        assert torch.equal(kc, kexp) and torch.equal(vc, vexp)


def _plant_ties(w, x, N, R, rows):
    """Make weight rows pairwise identical (exact logit ties) and aim rows[k]'s LayerNorm output at pair k % 3:
    a tie inside one tile, one across two tiles, one inside the last (partial) tile."""
    pairs = [(5 * R + 2, 5 * R + 9), (9 * R + R - 1, 10 * R), (N - 2, N - 1)]
    assert N % R and (N - 2) // R == (N - 1) // R == (N + R - 1) // R - 1     # the last tile is partial and holds the pair
    dirs = []
    for i, (a, z) in enumerate(pairs):
        v = torch.sign(torch.randn(w.shape[1], generator=torch.Generator(device=DEV).manual_seed(40 + i), device=DEV))
        w[a] = w[z] = (v * 4.0 / math.sqrt(w.shape[1])).to(torch.bfloat16)
        dirs.append(v)
    for k, r in enumerate(rows):
        x[r] = dirs[k % 3].to(torch.bfloat16)           # LayerNorm (weight 1, bias 0) keeps the direction
    return pairs


@pytest.mark.parametrize("B", [8, 16])
def test_gemv_ring_lm_head_argmax_partials(B):
    """Recombined partials (highest value, then lowest index) = the first argmax of the returned bf16 logits, with exact ties
    planted within a tile, across two tiles and in the last partial tile, on rows 0, 7, 8 and 15 (0, 7 and 4 for 8 rows)."""
    N, K = 49156, 2048
    g = torch.Generator(device=DEV).manual_seed(B)
    w, _ = _weights(N, K, g, bias=False)
    ln = (torch.ones(K, device=DEV).to(torch.bfloat16), torch.zeros(K, device=DEV).to(torch.bfloat16))
    x = torch.randn(B, K, generator=g, device=DEV).to(torch.bfloat16)
    nsm = _nsm()
    rpc = (N + nsm - 1) // nsm
    tpc = (rpc + 15) // 16
    R = (rpc + tpc - 1) // tpc
    rows = [0, 7, 8, 15] if B == 16 else [0, 7, 4]
    pairs = _plant_ties(w, x, N, R, rows)
    y, (val, idx) = E.op_gemv_ring(x, w, None, None, ln, epi=2)
    ref, scale, _ = _ring_ref(x, w, None, None, ln)
    _ring_check(y, ref, scale, f"lm_head B={B}")
    yc, val, idx = y.float().cpu(), val.cpu(), idx.cpu()
    nt = _lib.load().sv_op_ring_ntiles(N)
    assert val.shape[0] == nt == (N + R - 1) // R
    for r in range(B):
        v, i = val[:, r], idx[:, r]
        assert torch.equal(v, yc[r, i.long()]), r                 # every partial is a logit the kernel returned
        best = v.max()
        pick = int(i[v == best].min())
        assert pick == int(torch.argmax(yc[r])), (r, pick, int(torch.argmax(yc[r])))
    for k, r in enumerate(rows):
        a, z = pairs[k % len(pairs)]
        assert yc[r, a] == yc[r, z] == yc[r].max(), (r, a, z)   # the tie is real and is the maximum
        assert int(torch.argmax(yc[r])) == a
