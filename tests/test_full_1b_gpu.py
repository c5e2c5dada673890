"""Full-size StarVector-1B checks (BASELINE.json configs[1] dimensions): decode-mode equivalence and oracle parity."""
import os

import pytest
import torch

from oracle.pipeline import OracleStarVector
from parity import check_greedy_ids, oracle_greedy
from starvector_b200.config import dims_1b
from starvector_b200.engine import Engine, GenerationParams
from starvector_b200.weights import synthetic_images, synthetic_state_dict

pytestmark = pytest.mark.gpu
PROMPT = [44, 5678]


@pytest.fixture(scope="module")
def sd_1b():
    d = dims_1b(max_batch=2, max_len=1024)
    return d, synthetic_state_dict(d, seed=0)


_ORACLE = {}


def _oracle_fp32(d, sd):
    """ONE fp32 CPU oracle for the whole module (the weights do not depend on max_batch / max_len; building it costs ~20 s and
    4.4 GB).  fp32, not bf16: hosts without AMX emulate bf16 matmuls ~20x slower, and the tolerances below are stated against
    fp32 anyway (the bf16 oracle itself is ~0.05 max / 0.01 mean away from it)."""
    if "o" not in _ORACLE:
        torch.set_num_threads(min(32, os.cpu_count() or 1))   # as bench.py's CPU arm; with every logical CPU of the GPU box the 16-token B=8 oracle run took 250 s (8 s on 8 cores here)
        _ORACLE["o"] = OracleStarVector(d, sd, dtype=torch.float32, eos_token_id=None, pad_token_id=49152)
    return _ORACLE["o"]


def _engine(d, sd, **env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        e = Engine(d, 0)
    finally:
        for k, v in old.items():
            os.environ.pop(k, None) if v is None else os.environ.__setitem__(k, v)
    e.load_state_dict(sd)
    return e


def _gen(e, img, n, **kw):
    e.encode_images(img)
    e.prefill(torch.tensor([PROMPT] * img.shape[0]))
    return e.generate(GenerationParams(max_new_tokens=n, eos_token_id=None, pad_token_id=49152, **kw)).cpu()


def test_decode_modes_agree_1b(sd_1b):
    """Dataflow persistent kernel vs per-phase graph vs unfused kernels: same tokens, and logits within 2 bf16 ulp."""
    d, sd = sd_1b
    img = synthetic_images(d, 2, seed=1)
    outs, logits = {}, {}
    for name, env in (("mega", {"SV_FLOW": "1"}), ("graph", {"SV_FLOW": "0"}), ("legacy", {"SV_DECODE": "legacy"})):
        e = _engine(d, sd, **env)
        assert ("dataflow" in e.describe()) == (name == "mega"), e.describe()
        outs[name] = _gen(e, img, 40)
        e.encode_images(img)
        lg = [e.prefill(torch.tensor([PROMPT] * 2), return_logits=True)]
        for s in range(3):
            lg.append(e.decode_step(outs[name][:, s]))
        logits[name] = torch.stack(lg).cpu()
        if name == "mega":
            pen = _gen(e, img, 24, repetition_penalty=1.3)
            assert all(len(set(r.tolist())) > 1 for r in pen), "repetition penalty had no effect"
        e.close()
    assert torch.equal(outs["mega"], outs["graph"]) and torch.equal(outs["mega"], outs["legacy"])
    for k in ("graph", "legacy"):
        diff = (logits["mega"] - logits[k]).abs().max().item()
        assert diff < 0.1, (k, diff)


MARGIN_1B = 0.08        # logits; bf16 ulp at the top logit (~3.5) is 0.0156, the bf16 oracle's own max error vs fp32 is ~0.05


B8_ROWS = [0, 2, 5, 7]          # rows of the 8-image batch the CPU oracle recomputes (first, last and two in between)


def _oracle_b8(d, sd):
    """(images [8], ref_new [4, 16], ref_logits [16, 4, V]): the fp32 oracle's 16 greedy tokens for rows B8_ROWS of the 8-image
    batch, computed once per module -- the B = 8 test checks those rows of the engine's batch against it, the B = 1 test runs
    image 0 alone.  (On a busy GPU-box host the full 8-row oracle run alone took 250 s; the GPU suite has a time limit.)"""
    if "b8" not in _ORACLE:
        img = synthetic_images(d, 8, seed=2)
        ref_new, ref_logits = oracle_greedy(_oracle_fp32(d, sd), img[B8_ROWS].float(), PROMPT, (), 16)
        _ORACLE["b8"] = (img, ref_new, ref_logits)
    return _ORACLE["b8"]


def test_1b_matches_cpu_oracle(sd_1b):
    """B = 1 (the headline shape): prefill logits + 6 greedy ids of the full-size model against the CPU oracle (reference
    modules + HF), re-synced by teacher forcing after a tolerated flip."""
    d, sd = sd_1b
    img8, ref_new, ref_logits = _oracle_b8(d, sd)
    img = img8[:1]                                             # image 0 = oracle row 0
    e = _engine(d, sd)
    e.encode_images(img)
    lg = e.prefill(torch.tensor([PROMPT]), return_logits=True).cpu()
    got = e.generate(GenerationParams(max_new_tokens=6, eos_token_id=None, pad_token_id=49152)).cpu().long()
    e.close()
    o = _oracle_fp32(d, sd)
    err = (lg[0] - ref_logits[0, 0]).abs()
    assert err.max().item() < 0.25 and err.mean().item() < 0.03, (err.max().item(), err.mean().item())
    check_greedy_ids(got, ref_new[:1, :6], ref_logits[:6, :1], MARGIN_1B, lambda ids: o.teacher_forced_logits(img.float(), PROMPT, ids))


def test_1b_batch8_greedy_vs_oracle(sd_1b):
    """B = 8 rows at full 1B dims (the per-GPU slice of BASELINE configs[2]): the engine runs all 8 images; prefill logits and 16
    greedy tokens of rows 0 / 2 / 5 / 7 against the fp32 CPU oracle (bf16 matmuls are emulated and ~20x slower on hosts without
    AMX), re-synced by teacher forcing after a tolerated flip."""
    d, sd = dims_1b(max_batch=8, max_len=512), sd_1b[1]
    img, ref_new, ref_logits = _oracle_b8(d, sd)
    e = _engine(d, sd)
    e.encode_images(img)
    lg = e.prefill(torch.tensor([PROMPT] * 8), return_logits=True).cpu()
    got = e.generate(GenerationParams(max_new_tokens=16, eos_token_id=None, pad_token_id=49152)).cpu().long()
    e.close()
    assert got.shape == (8, 16) and lg.shape[0] == 8
    o = _oracle_fp32(d, sd)
    err = (lg[B8_ROWS] - ref_logits[0]).abs()
    assert err.max().item() < 0.25 and err.mean().item() < 0.03, (err.max().item(), err.mean().item())
    check_greedy_ids(got[B8_ROWS], ref_new, ref_logits, MARGIN_1B,
                     lambda ids: o.teacher_forced_logits(img[B8_ROWS].float(), PROMPT, ids))


class _CountingEngine:
    """The host-stepped beam loop over the engine, counting the steps whose cache permutation is not the identity."""

    def __init__(self, eng):
        self._eng, self.dims, self.steps, self.reordered = eng, eng.dims, 0, 0

    def encode_images(self, image):
        return self._eng.encode_images(image)

    def prefill(self, prompt_ids, return_logits=False):
        return self._eng.prefill(prompt_ids, return_logits=return_logits)

    def reorder_cache(self, idx):
        self.steps += 1
        self.reordered += int(not torch.equal(idx.cpu().long(), torch.arange(idx.numel())))
        return self._eng.reorder_cache(idx)

    def decode_step(self, tokens):
        return self._eng.decode_step(tokens)


def test_1b_device_beam_search_equals_host_loop(sd_1b):
    """sv_beam_search at the 1B shape (24 layers, 49156-token vocabulary, the whole search in the replayed graph) against the
    host-stepped loop over the same engine: the reference configuration (2 images, num_beams=2, early_stopping=True) and 4
    images x 4 beams (16 cache rows).  An untied random lm_head makes the beams reorder at most steps."""
    from starvector_b200.beam_search import beam_search
    from test_beam_gpu import PROMPT as BEAM_PROMPT, _same_or_equivalent

    d, sd = dims_1b(max_batch=16, max_len=512), dict(sd_1b[1])
    g = torch.Generator().manual_seed(3)
    head = (torch.randn(d.vocab, d.hidden, generator=g) * 0.2).to(torch.bfloat16)
    sd["model.svg_transformer.transformer.lm_head.weight"] = head
    e = _engine(d, sd)
    pad = 49152
    try:
        for B, nb in ((2, 2), (4, 4)):
            img = synthetic_images(d, B, seed=4 + B)
            ids = torch.tensor([BEAM_PROMPT] * B)
            kw = dict(num_beams=nb, max_new_tokens=32, early_stopping=True, eos_token_id=0, pad_token_id=pad)
            host = _CountingEngine(e)
            ref = beam_search(host, img, ids, impl="host", **kw).cpu()
            assert host.reordered * 2 > host.steps, (B, nb, host.reordered, host.steps)
            got = beam_search(e, img, ids, impl="device", **kw).cpu()
            assert got.shape == ref.shape, (B, nb, got.shape, ref.shape)
            if not torch.equal(got, ref):
                o = _oracle_fp32(d, sd_1b[1])
                tied = o.llm.lm_head.weight
                o.llm.lm_head.weight = torch.nn.Parameter(head.float())
                try:
                    _same_or_equivalent(o, img.float(), got, ref, pad, 1.0, 1.0)
                finally:
                    o.llm.lm_head.weight = tied
    finally:
        e.close()


@pytest.mark.parametrize("mode", ["flow", "graph"])
def test_1b_long_context_logits(sd_1b, mode):
    """The benchmarked shape: 4096 new tokens at B = 1 reach context 4355.  Teacher-force 4100 fixed tokens and compare the
    next-token logits at contexts ~600 / ~1800 / ~4300 with the fp32 oracle's full forward (attention over 3 / 8 / 17
    key splits in the dataflow kernel, 2 / 4 / 8-CTA clusters in the per-phase graph path)."""
    d, sd = dims_1b(max_batch=1, max_len=4500), sd_1b[1]
    img = synthetic_images(d, 1, seed=1)
    n_forced = 4100
    g = torch.Generator().manual_seed(7)
    forced = torch.randint(0, 49152, (1, n_forced), generator=g)
    steps = [340, 1540, 4040]                      # generated-token index j: context = 259 + j
    e = _engine(d, sd, SV_FLOW="1" if mode == "flow" else "0")
    assert ("dataflow" in e.describe()) == (mode == "flow"), e.describe()
    e.encode_images(img)
    e.prefill(torch.tensor([PROMPT]))
    got = {}
    for j in range(n_forced):
        lg = e.decode_step(forced[:, j], return_logits=(j + 1) in steps)
        if (j + 1) in steps:
            got[j + 1] = lg.float().cpu()
    e.close()
    if "long_ref" not in _ORACLE:          # one oracle forward over the 4359 tokens serves both decode modes
        _ORACLE["long_ref"] = _oracle_fp32(d, sd).teacher_forced_logits_at(img.float(), PROMPT, forced, steps)         # [1, 3, V]
    ref = _ORACLE["long_ref"]
    for k, j in enumerate(steps):
        err = (got[j][0] - ref[0, k]).abs()
        # same bound as the prefill logits: the bf16 oracle itself is ~0.05 max / 0.01 mean away from fp32
        assert err.max().item() < 0.25 and err.mean().item() < 0.03, (mode, j, err.max().item(), err.mean().item())
        assert ref[0, k].argmax().item() == got[j][0].argmax().item() or \
            (ref[0, k].max() - ref[0, k][got[j][0].argmax()]).item() < MARGIN_1B, (mode, j)
