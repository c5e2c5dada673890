"""Launches per replayed decode step: every generation loop adds exactly the kernels of its step graph, once per step.

The expected counts follow from the kernel list of one step of a v1 model with L layers (no RoPE):
* fused chain: per layer the c_attn ring GEMV (LayerNorm and KV append fused), the cluster attention and the c_proj, c_fc
  and c_fc2 ring GEMVs, 5L; then the lm_head ring GEMV with ln_f fused, 1.  Sampling embeds the selected token first, 1.
* per-op chain: the token embedding, per layer LayerNorm, c_attn, KV append, split and merge attention, c_proj, LayerNorm,
  c_fc and c_fc2, 9L; then ln_f and lm_head, 2.
* selection: greedy on the fused chain is select_fused alone (it embeds the next input); otherwise the greedy or sampling
  kernel and gen_finalize.  A session step selects with one kernel, the per-row variant.
* beam bookkeeping: candidates, beam step and the two-launch KV suffix copy, 4.
Each count is the difference between two runs that differ by k steps only, so the launches around the loop cancel.  EOS
is off, so every step of the budget runs."""
import os

import pytest
import torch

from starvector_b200.config import dims_tiny
from starvector_b200.engine import Engine, GenerationParams
from starvector_b200.weights import synthetic_images, synthetic_state_dict

pytestmark = pytest.mark.gpu

PROMPT = [44, 78]
L = 3
N, K = 8, 5                 # runs of N and N + K steps; N + K stays below the poll interval of the beam loop


@pytest.fixture(scope="module")
def setup():
    d = dims_tiny(max_batch=4, n_layer=L)
    sd = synthetic_state_dict(d, seed=0, init="randomized")
    engines = {}
    for mode, env in (("fused", None), ("legacy", "legacy")):
        if env:
            os.environ["SV_DECODE"] = env
        try:
            eng = Engine(d, 0)
        finally:
            os.environ.pop("SV_DECODE", None)
        eng.load_state_dict(sd)
        engines[mode] = eng
    assert "ring-gemv-graph" in engines["fused"].describe() and "legacy-kernels" in engines["legacy"].describe()
    yield d, engines, synthetic_images(d, 2, seed=1)
    for eng in engines.values():
        eng.close()


def _launches(eng, run):
    c0 = eng.launch_count()
    run()
    return eng.launch_count() - c0


def _generate(d, eng, img, n, stream=False, **kw):
    eng.encode_images(img)
    eng.prefill(torch.tensor([PROMPT] * img.shape[0]))
    p = GenerationParams(max_new_tokens=n, eos_token_id=None, pad_token_id=d.vocab - 4, poll_interval=4, **kw)
    chunks, out = [], []
    on_tokens = (lambda ids, first_step: chunks.append(ids)) if stream else None
    count = _launches(eng, lambda: out.append(eng.generate(p, on_tokens=on_tokens)))
    assert out[0].shape == (img.shape[0], n)
    if stream:
        assert torch.equal(torch.cat(chunks, dim=1), out[0].cpu())
    return count


@pytest.mark.parametrize("mode,kw,per_step", [
    ("fused", dict(), 5 * L + 2),
    ("fused", dict(stream=True), 5 * L + 2),
    ("fused", dict(do_sample=True, seed=3), 5 * L + 4),
    ("legacy", dict(), 9 * L + 5),
    ("legacy", dict(do_sample=True, seed=3), 9 * L + 5),
], ids=["fused-greedy", "fused-greedy-stream", "fused-sample", "legacy-greedy", "legacy-sample"])
def test_generate_launches_per_step(setup, mode, kw, per_step):
    d, engines, img = setup
    eng = engines[mode]
    assert _generate(d, eng, img, N + K, **kw) - _generate(d, eng, img, N, **kw) == K * per_step


@pytest.mark.parametrize("mode,per_step", [("fused", 5 * L + 1 + 4), ("legacy", 9 * L + 3 + 4)], ids=["fused", "legacy"])
def test_beam_search_launches_per_step(setup, mode, per_step):
    d, engines, img = setup
    eng, nb = engines[mode], 2

    def search(n):
        eng.encode_images(img.repeat_interleave(nb, dim=0))
        eng.prefill(torch.tensor([PROMPT] * (img.shape[0] * nb)))
        return _launches(eng, lambda: eng.beam_search_device(img.shape[0], num_beams=nb, max_new_tokens=n,
                                                             early_stopping="never", eos_token_id=None,
                                                             pad_token_id=d.vocab - 4))

    assert search(N + K) - search(N) == K * per_step


@pytest.mark.parametrize("mode,per_step", [("fused", 5 * L + 2), ("legacy", 9 * L + 4)], ids=["fused", "legacy"])
def test_session_run_launches_per_step(setup, mode, per_step):
    d, engines, img = setup
    eng = engines[mode]
    eng.session_begin(GenerationParams(max_new_tokens=4 * (N + K), eos_token_id=None, pad_token_id=d.vocab - 4), slots=2)
    try:
        eng.session_admit(img, torch.tensor([PROMPT] * 2), [0, 1])
        counts = []
        for n in (N, N + K):
            res = []
            counts.append(_launches(eng, lambda: res.append(eng.session_run(n))))
            steps, finished, _ = res[0]
            assert steps == n and not any(finished)
    finally:
        eng.session_end()
    assert counts[1] - counts[0] == K * per_step
    assert counts[0] == N * per_step            # a session run launches nothing but its replays
