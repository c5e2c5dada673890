"""Continuous batching: many images through a fixed set of cache rows ("slots"), refilled as rows finish.

The engine decodes up to `max_batch` rows per weight stream, and a step costs about the same whether 1 or 16 rows use
it.  Running a large workload as groups of `max_batch` rows makes every group as long as its longest member.  A session
(`sv_session_*`) instead lets every row finish on its own: its tokens are harvested, the next queued image is encoded
and prefilled into that slot while the other slots keep their caches, and the replayed decode graph continues.

`ContinuousScheduler` is the host side: a FIFO queue of requests and a free-slot list.  It only talks to the engine
through `session_begin / session_admit / session_run / session_read / session_end` (beam sessions: `beam_session_begin /
beam_session_admit` and the same run / read / end), so it can be driven by a stand-in engine on a machine without a GPU.
With `num_beams > 1` the unit of admission is a group of `num_beams` contiguous slots that runs one image's beam search.
"""
from __future__ import annotations

import collections
import time
from typing import Callable, List, Optional, Sequence

import torch


def spec_session_k(params, slots: int, engine) -> int:
    """Drafts per row a session with these parameters speculates with: `params.prompt_lookup_num_tokens` clamped to
    `slots - 1` on v1 engines on the fused decode path, 0 (a plain session) without the hint, with one slot, on v2
    (StarVector-8B) engines or with `SV_DECODE=legacy`.  Inside a session the hint changes the speed only."""
    k = int(getattr(params, "prompt_lookup_num_tokens", 0) or 0)
    if k <= 0 or slots < 2 or engine.dims.variant != 0 or not engine.fused_decode:
        return 0
    return min(k, slots - 1)


class ContinuousScheduler:
    """Runs requests (one image each, `n` completions per image) through a decode session of `slots` cache rows.

    Every completion gets the tokens a one-image `generate` with the same parameters and its own seed gives, up to and
    including its EOS / stop sequence, or `max_new_tokens[i]` tokens.  After `run`, `stats` holds the decode steps, the
    number of admissions, the host wall time spent in admission (encode + prefill) and in decoding, and `admit_step`: for
    every completion, the number of decode steps the session had run when it was admitted (while two rows decode side
    by side, their context lengths differ by the difference of their admit steps).  A speculative session
    (`spec_session_k`) adds `spec`: its verify steps, drafts proposed and drafts accepted; `steps` then counts verify
    steps."""

    def __init__(self, engine, slots: Optional[int] = None, num_beams: int = 1):
        self.engine = engine
        self.slots = int(slots if slots is not None else engine.dims.max_batch)
        self.num_beams = int(num_beams)
        if not 1 <= self.slots <= engine.dims.max_batch:
            raise ValueError(f"slots {self.slots} outside [1, {engine.dims.max_batch}]")
        if self.num_beams < 1 or self.slots % self.num_beams:
            raise ValueError(f"slots {self.slots} must be a multiple of num_beams {self.num_beams}")
        self.stats = {}

    def run(self, pixels: torch.Tensor, prompt_ids: torch.Tensor, params, *, max_new_tokens: Optional[Sequence[int]] = None,
            seeds: Optional[Sequence[int]] = None, n: int = 1,
            on_finish: Optional[Callable[[int, torch.Tensor], None]] = None) -> List[torch.Tensor]:
        """pixels `[N, 3, S, S]`; prompt_ids `[P]` (shared) or `[N, P]`; params: the session's `GenerationParams` (its
        `max_new_tokens` is the session cap).  `max_new_tokens`: one cap per image, each in [1, params.max_new_tokens].
        `seeds`: one per completion (default `params.seed + k` for completion k = i * n + j).  Returns one int32 tensor per
        completion, in request order (index i * n + j); `on_finish(index, ids)` is called as each one completes.
        With `num_beams > 1`, params is a `BeamSearchParams` of that width and every image is one request (n = 1) whose
        result is its best hypothesis."""
        N = int(pixels.shape[0])
        n = int(n)
        cap = int(params.max_new_tokens)
        nb = self.num_beams
        if nb > 1 and (n != 1 or int(params.num_beams) != nb):
            raise ValueError(f"a beam session of width {nb} takes one request per image and params with num_beams = {nb}")
        if n < 1 or n > self.slots:
            raise ValueError(f"n = {n} completions per image must be in [1, {self.slots}] (the session's slots)")
        if prompt_ids.dim() == 1:
            prompt_ids = prompt_ids.unsqueeze(0).expand(N, -1)
        if prompt_ids.dim() != 2 or prompt_ids.shape[0] != N:
            raise ValueError("prompt_ids must be [P] or [N, P]")
        caps = [cap] * N if max_new_tokens is None else [int(m) for m in max_new_tokens]
        if len(caps) != N:
            raise ValueError(f"max_new_tokens has {len(caps)} entries for {N} images")
        for i, m in enumerate(caps):
            if not 1 <= m <= cap:
                raise ValueError(f"max_new_tokens[{i}] = {m} outside [1, {cap}] (the session cap, params.max_new_tokens)")
        seeds = [int(params.seed) + k for k in range(N * n)] if seeds is None else [int(s) for s in seeds]
        if len(seeds) != N * n:
            raise ValueError(f"seeds has {len(seeds)} entries for {N * n} completions")

        eng = self.engine
        queue = collections.deque(range(N))
        free = list(range(0, self.slots, nb))       # free units: slots, or the first slots of free beam groups
        owner = {}                                   # (first) slot -> completion index
        results: List[Optional[torch.Tensor]] = [None] * (N * n)
        admit_step = [0] * (N * n)
        steps = admissions = 0
        t_admit = t_decode = 0.0
        spec = nb == 1 and spec_session_k(params, self.slots, eng) > 0
        spec_stats = None
        if nb > 1:
            eng.beam_session_begin(params, self.slots)
        else:
            eng.session_begin(params, self.slots)
        try:
            while queue or owner:
                # FIFO admission: as many queued images as there are free units for all their completions
                batch = []
                while queue and len(free) >= n:
                    i = queue.popleft()
                    batch.append((i, [free.pop(0) for _ in range(n)]))
                if batch:
                    imgs = [i for i, _ in batch]
                    slots, src, mx, sd = [], [], [], []
                    for b, (i, sl) in enumerate(batch):
                        for j, s in enumerate(sl):
                            slots.append(s); src.append(b); mx.append(caps[i]); sd.append(seeds[i * n + j])
                            owner[s] = i * n + j
                            admit_step[i * n + j] = steps
                    t0 = time.perf_counter()
                    if nb > 1:
                        eng.beam_session_admit(pixels[imgs], prompt_ids[imgs], [s // nb for s in slots], max_new_tokens=mx,
                                               seeds=sd)
                    else:
                        eng.session_admit(pixels[imgs], prompt_ids[imgs], slots, max_new_tokens=mx, seeds=sd, src=src)
                    t_admit += time.perf_counter() - t0
                    admissions += 1
                t0 = time.perf_counter()
                ran, finished, _lens = eng.session_run(cap)
                t_decode += time.perf_counter() - t0
                steps += ran
                done = [s for s in range(self.slots) if finished[s]]
                if not done and ran == 0:
                    raise RuntimeError("decode session made no progress (no slot finished and no step ran)")
                for s in done:
                    k = owner.pop(s)
                    ids = eng.session_read(s)
                    results[k] = ids
                    free.append(s)
                    if on_finish is not None:
                        on_finish(k, ids)
                free.sort()
            if spec:
                spec_stats = eng.session_spec_stats()
        finally:
            eng.session_end()
        self.stats = {"steps": steps, "admissions": admissions, "admit_s": t_admit, "decode_s": t_decode,
                      "admit_step": admit_step}
        if spec_stats is not None:
            self.stats["spec"] = spec_stats
        return results
