"""Tokenizer plumbing for the facade.

The reference builds its tokenizer from the hub (`AutoTokenizer.from_pretrained`,
llm/starcoder.py:40-53: +[PAD] +`<svg-start>`,`<image-start>`,`<caption-start>`).  Offline there
are no tokenizer files, so synthetic models use `SyntheticTokenizer`: a deterministic,
reversible id<->text stand-in that keeps the attributes/call shapes the reference code touches
(`pad_token_id`, `eos_token_id`, `__call__(...)['input_ids']`, `batch_decode`).  With a local
checkpoint directory that has tokenizer files, `load_tokenizer` returns the real one, prepared
exactly as the reference does.
"""
from __future__ import annotations

import re
from typing import Dict, List, Sequence, Union


class SyntheticTokenizer:
    """ids 0..vocab-1; text form of id k is ``<t{k}>``; '<svg' / '</svg>' have fixed multi-token ids."""

    def __init__(self, vocab_size: int, n_added: int = 4):
        self.vocab_size = vocab_size
        self.eos_token_id = 0
        self.bos_token_id = 0
        self.pad_token_id = vocab_size - n_added          # '[PAD]' is the first added token (starcoder.py:47-48)
        self.eos_token = "<|endoftext|>"
        self.pad_token = "[PAD]"
        self.padding_side = "right"
        base = max(vocab_size - n_added, 8)
        self._known: Dict[str, List[int]] = {
            "<svg": [44 % base or 1, 5678 % base or 2],
            "</svg>": [1245 % base or 3, 7 % base or 4, 29 % base or 5],
        }
        self._special = {self.eos_token_id, self.pad_token_id}
        self._named = {self.eos_token: self.eos_token_id, self.pad_token: self.pad_token_id}
        if n_added >= 5:                                  # v2 (llm/starcoder2.py:45-50): <svg-end> is the 4th token after [PAD]
            self._named["<svg-end>"] = self.pad_token_id + 4

    def __len__(self) -> int:
        return self.vocab_size

    def encode(self, text: str, add_special_tokens: bool = False) -> List[int]:
        if text in self._known:
            return list(self._known[text])
        ids: List[int] = []
        named = "".join(re.escape(k) + "|" for k in self._named)
        for m in re.finditer(r"<t(\d+)>|" + named + r"<svg|</svg>|\S+", text):
            tok = m.group(0)
            if tok in self._named:
                ids.append(self._named[tok])
            elif m.group(1) is not None:
                ids.append(int(m.group(1)) % self.vocab_size)
            elif tok in self._known:
                ids.extend(self._known[tok])
            else:
                ids.append(1 + (sum(tok.encode()) * 2654435761 % (self.pad_token_id - 1)))
        return ids

    def __call__(self, text: Union[str, Sequence[str]], add_special_tokens: bool = True, return_tensors=None, **kw):
        single = isinstance(text, str)
        rows = [self.encode(t) for t in ([text] if single else text)]
        if kw.get("truncation") and kw.get("max_length") is not None:
            rows = [r[: int(kw["max_length"])] for r in rows]
        if single and return_tensors is None:
            return {"input_ids": rows[0], "attention_mask": [1] * len(rows[0])}
        width = max(len(r) for r in rows)
        ids = [r + [self.pad_token_id] * (width - len(r)) for r in rows]
        mask = [[1] * len(r) + [0] * (width - len(r)) for r in rows]
        if return_tensors == "pt":
            import torch

            return {"input_ids": torch.tensor(ids, dtype=torch.long), "attention_mask": torch.tensor(mask, dtype=torch.long)}
        return {"input_ids": ids, "attention_mask": mask}

    def decode(self, ids, skip_special_tokens: bool = True) -> str:
        ids = [int(i) for i in ids]
        out, i = [], 0
        known = sorted(self._known.items(), key=lambda kv: -len(kv[1]))
        while i < len(ids):
            for text, seq in known:
                if ids[i:i + len(seq)] == seq:
                    out.append(text)
                    i += len(seq)
                    break
            else:
                if not (skip_special_tokens and ids[i] in self._special):
                    out.append(f"<t{ids[i]}>")
                i += 1
        return "".join(out)

    def batch_decode(self, batch, skip_special_tokens: bool = True) -> List[str]:
        rows = batch.tolist() if hasattr(batch, "tolist") else batch
        return [self.decode(r, skip_special_tokens) for r in rows]


def load_tokenizer(path_or_none, vocab_size: int, v2: bool = False):
    """Real tokenizer when a local directory provides one, prepared as the reference does — v1: llm/starcoder.py:40-53
    (fast tokenizer, + [PAD], + 3 added tokens); v2: llm/starcoder2.py:36-53 (`use_fast=False`, + 4 added tokens incl.
    `<svg-end>`, `padding_side = "left"`) — else the synthetic stand-in (3 / 4 added tokens after [PAD])."""
    import os

    if path_or_none and os.path.isdir(path_or_none) and any(
            os.path.exists(os.path.join(path_or_none, f)) for f in ("tokenizer.json", "vocab.json", "tokenizer_config.json")):
        from transformers import AutoTokenizer

        if v2:
            try:
                tok = AutoTokenizer.from_pretrained(path_or_none, local_files_only=True, use_fast=False)
            except (OSError, ValueError):           # a directory that only ships tokenizer.json has no slow tokenizer
                tok = AutoTokenizer.from_pretrained(path_or_none, local_files_only=True)
        else:
            tok = AutoTokenizer.from_pretrained(path_or_none, local_files_only=True)
        if tok.eos_token_id is None:
            tok.add_special_tokens({"eos_token": "[EOS]"})
        if tok.pad_token_id is None:
            tok.add_special_tokens({"pad_token": "[PAD]"})
        if v2:
            tok.add_tokens(["<svg-start>", "<image-start>", "<caption-start>", "<svg-end>"])
            tok.padding_side = "left"
        else:
            tok.add_tokens(["<svg-start>", "<image-start>", "<caption-start>"])
        return tok
    tok = SyntheticTokenizer(vocab_size, n_added=5 if v2 else 4)
    if v2:
        tok.padding_side = "left"
    return tok
