"""Greedy-id parity contract shared by the GPU tests (DESIGN.md "Numerics contract", SURVEY.md §7 hard part (a)).

The engine and the CPU oracle accumulate in different orders, so two logits closer than a few bf16 ulp may swap.
The contract therefore is:

1. wherever engine and oracle ids agree nothing more is asked;
2. at the first disagreement of a row, the oracle's own top-1/top-2 margin at that step must be below ``tol``;
3. the comparison then RE-SYNCS by teacher forcing: the oracle is run once over the ENGINE's sequence, and at every later
   step the engine's token must be the oracle's argmax for that history or lie within ``tol`` of it.  A wrong KV cache,
   a mis-merged attention partial or a bad position therefore still fails after a tolerated flip.

Rows stop being checked after they emitted EOS (HF pads them) and after a stop sequence ended the batch.
"""
from typing import Optional, Sequence

import torch


def _penalised(row: torch.Tensor, seen: set, repetition_penalty: float) -> torch.Tensor:
    """HF RepetitionPenaltyLogitsProcessor on one fp32 logits row: the scores greedy selection compares."""
    row = row.clone()
    if repetition_penalty != 1.0 and seen:
        idx = torch.tensor(sorted(seen))
        v = row[idx]
        row[idx] = torch.where(v < 0, v * repetition_penalty, v / repetition_penalty)
    return row


def check_greedy_ids(got: torch.Tensor, ref_new: torch.Tensor, ref_logits: torch.Tensor, tol: float, teacher_forced,
                     eos_token_id: Optional[int] = None, repetition_penalty: float = 1.0) -> dict:
    """got / ref_new: [B, n] generated ids (engine / oracle).  ref_logits: [n_ref, B, V] raw fp32 logits of the oracle
    (before the repetition penalty, which is applied here to the ids generated so far).  teacher_forced(ids[B, n]) ->
    [B, n + 1, V] fp32 oracle logits under the engine's history (called at most once).
    Returns counters for the caller's own asserts ("flips": tolerated disagreements, "resynced": steps checked by (3))."""
    got = got.cpu().long()
    ref_new = ref_new.cpu().long()
    B, n = got.shape
    stats = {"flips": 0, "resynced": 0}
    if got.shape == ref_new.shape and torch.equal(got, ref_new):
        return stats
    tf = None
    for b in range(B):
        n_cmp = min(n, ref_new.shape[1])
        first = next((s for s in range(n_cmp) if got[b, s] != ref_new[b, s]), None)
        if first is None:
            continue
        seen = set(int(t) for t in got[b, :first].tolist())
        top2 = _penalised(ref_logits[first, b].float(), seen, repetition_penalty).topk(2).values
        margin = (top2[0] - top2[1]).item()
        assert margin < tol, f"row {b} step {first}: ids differ ({int(got[b, first])} vs {int(ref_new[b, first])}) at oracle margin {margin:.4f}"
        stats["flips"] += 1
        if tf is None:
            tf = teacher_forced(got).float()                       # [B, n + 1, V]
        for s in range(first, n):
            tok = int(got[b, s])
            if eos_token_id is not None and s > 0 and int(got[b, s - 1]) == eos_token_id:
                break                                              # finished row: the rest is padding
            row = _penalised(tf[b, s], seen, repetition_penalty)
            gap = (row.max() - row[tok]).item()
            assert gap < tol, f"row {b} step {s} (after the flip at {first}): engine token {tok} is {gap:.4f} below the oracle's best for the engine's own history"
            stats["resynced"] += 1
            seen.add(tok)
    if stats["flips"] == 0:
        assert got.shape == ref_new.shape, (got.shape, ref_new.shape)     # same ids up to the shorter length but another length
    return stats


def oracle_greedy(oracle, img, prompt: Sequence[int], stop_ids: Sequence[int], n_new: int, **kw):
    """(ref_new [B, n], ref_logits [n, B, V]) of the reference path run greedily (num_beams=1)."""
    ref, ref_logits = oracle.generate_im2svg_ids(img, prompt, stop_ids, return_logits=True, use_nucleus_sampling=False, num_beams=1,
                                                 max_length=oracle.dims.query_length + len(prompt) + n_new, **kw)
    return ref[:, len(prompt):], ref_logits
