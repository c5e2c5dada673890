"""`Engine`: the thin object around one `sv_engine*` (one model replica on one GPU).

PyTorch is used only for device memory, dtype views and the current stream handle; all
compute happens inside libstarvector_b200.so.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import threading
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import torch

from . import _lib
from .config import ModelDims

_DTYPES = {torch.bfloat16: _lib.SV_DTYPE_BF16, torch.float32: _lib.SV_DTYPE_F32, torch.float16: _lib.SV_DTYPE_F16}


@dataclasses.dataclass
class GenerationParams:
    """HF `generate()` kwargs after the reference's whitelist (starvector_base.py:223-241)."""

    max_new_tokens: int
    do_sample: bool = False
    temperature: float = 1.0
    top_p: float = 1.0
    repetition_penalty: float = 1.0
    eos_token_id: Optional[int] = 0
    pad_token_id: int = 0
    stop_ids: Sequence[int] = ()
    stop_row0_only: bool = True
    seed: int = 0
    poll_interval: int = 16
    # prompt-lookup speculative decoding (HF `prompt_lookup_num_tokens` / `max_matching_ngram_size`): > 0 drafts up to that
    # many tokens per step from n-gram matches in the generated tokens (`sv_generate_speculative`); the tokens are the same
    prompt_lookup_num_tokens: int = 0
    max_matching_ngram_size: int = 2

    def to_c(self) -> _lib.GenParams:
        if len(self.stop_ids) > 8:
            raise ValueError("stop sequence longer than 8 tokens")
        p = _lib.GenParams()
        p.max_new_tokens = int(self.max_new_tokens)
        p.do_sample = int(bool(self.do_sample))
        p.temperature = float(self.temperature)
        p.top_p = float(self.top_p)
        p.repetition_penalty = float(self.repetition_penalty)
        p.eos_token_id = -1 if self.eos_token_id is None else int(self.eos_token_id)
        p.pad_token_id = int(self.pad_token_id)
        p.n_stop_ids = len(self.stop_ids)
        for i, s in enumerate(self.stop_ids):
            p.stop_ids[i] = int(s)
        p.stop_row0_only = int(bool(self.stop_row0_only))
        p.seed = int(self.seed) & (2 ** 64 - 1)
        p.poll_interval = int(self.poll_interval)
        return p


@dataclasses.dataclass
class BeamSearchParams:
    """HF `generate(num_beams > 1)` kwargs as `sv_beam_search` and beam sessions take them.  `pad_token_id` is the fill of
    the sequence rows (HF: pad if given, else eos; -1 without EOS), as `beam_search` passes it."""

    num_beams: int
    max_new_tokens: int
    do_sample: bool = False
    temperature: float = 1.0
    top_p: float = 1.0
    repetition_penalty: float = 1.0
    length_penalty: float = 1.0
    early_stopping: object = True            # True, False or "never"
    eos_token_id: Optional[int] = 0
    pad_token_id: int = 0
    stop_ids: Sequence[int] = ()
    seed: int = 0
    poll_interval: int = 16

    def to_c(self) -> _lib.BeamParams:
        if len(self.stop_ids) > 8:
            raise ValueError("stop sequence longer than 8 tokens")
        bp = _lib.BeamParams()
        bp.num_beams, bp.max_new_tokens, bp.do_sample = int(self.num_beams), int(self.max_new_tokens), int(bool(self.do_sample))
        bp.early_stopping = 2 if self.early_stopping == "never" else int(self.early_stopping is True)
        bp.temperature, bp.top_p = float(self.temperature), float(self.top_p)
        bp.repetition_penalty, bp.length_penalty = float(self.repetition_penalty), float(self.length_penalty)
        bp.eos_token_id = -1 if self.eos_token_id is None else int(self.eos_token_id)
        bp.pad_token_id = int(self.pad_token_id)
        bp.n_stop_ids = len(self.stop_ids)
        for i, t in enumerate(self.stop_ids):
            bp.stop_ids[i] = int(t)
        bp.poll_interval = int(self.poll_interval)
        bp.seed = int(self.seed) & (2 ** 64 - 1)
        return bp


def _stream_ptr(device: torch.device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class Engine:
    def __init__(self, dims: ModelDims, device: int | torch.device = 0):
        self._lib = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.EngineError("starvector_b200: no CUDA device visible; this engine has no CPU fallback")
        self.device = torch.device("cuda", device if isinstance(device, int) else (device.index or 0))
        self.dims = dims
        desc = _lib.ModelDesc(
            variant=dims.variant, image_size=dims.image_size, patch_size=dims.patch_size, vit_width=dims.vit_width,
            vit_layers=dims.vit_layers, vit_heads=dims.vit_heads, vit_mlp=dims.vit_mlp, adapter_norm=dims.adapter_norm,
            hidden=dims.hidden, n_layer=dims.n_layer, n_head=dims.n_head, n_kv_head=dims.n_kv_head,
            head_dim=dims.head_dim, n_inner=dims.n_inner, n_positions=dims.n_positions, vocab=dims.vocab,
            ln_eps=dims.ln_eps, max_batch=dims.max_batch, max_len=dims.max_len,
            rope_theta=dims.rope_theta, sliding_window=dims.sliding_window, vit_ln_eps=dims.vit_ln_eps,
        )
        h = C.c_void_p()
        torch.cuda.init()
        torch.zeros(1, device=self.device)        # make sure the primary context exists
        _lib.check(self._lib, self._lib.sv_engine_create(C.byref(desc), self.device.index, C.byref(h)))
        self._h = h
        self._lock = threading.Lock()             # engine is not re-entrant (SURVEY.md §3.3: threaded callers)
        self.query_length = dims.query_length
        self._batch = 0
        self._prompt_len = 0

    # -- lifecycle -----------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.sv_engine_destroy(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, code: int) -> None:
        _lib.check(self._lib, code, self._h)

    # -- weights -------------------------------------------------------------------------
    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True) -> None:
        """Copy a reference-named state dict (CPU or CUDA tensors; bf16/fp16/fp32) into the engine."""
        wte_key = ("model.svg_transformer.transformer.model.embed_tokens.weight" if self.dims.variant == 1
                   else "model.svg_transformer.transformer.transformer.wte.weight")
        lm_key = "model.svg_transformer.transformer.lm_head.weight"
        with self._lock:
            for name, t in sd.items():
                if name == lm_key and wte_key in sd and (t is sd[wte_key] or t.data_ptr() == sd[wte_key].data_ptr()
                                                          or torch.equal(t, sd[wte_key])):
                    continue                       # tied head: the engine aliases wte
                if not t.is_floating_point():
                    continue
                if t.dtype not in _DTYPES:
                    t = t.float()
                t = t.contiguous()
                shape = (C.c_int64 * max(t.dim(), 1))(*t.shape)
                code = self._lib.sv_engine_load_weight(self._h, name.encode(), C.c_void_p(t.data_ptr()), shape,
                                                       t.dim(), _DTYPES[t.dtype])
                if code == _lib.SV_ERR_INVALID and not strict:
                    continue
                self._ck(code)
            if self.dims.variant == 1:
                self._load_rope_tables()
            missing = self._lib.sv_engine_missing_weights(self._h)
            if missing and strict:
                names = self._lib.sv_last_error(self._h).decode()
                raise KeyError(f"{missing} weights missing from state dict, e.g. {names.splitlines()[:4]}")

    def _load_rope_tables(self) -> None:
        """cos/sin tables computed exactly as Starcoder2RotaryEmbedding does (fp32 outer product, cast to bf16), so the
        engine's RoPE inputs are bit-identical to the reference's; the engine's own on-device table is the fallback."""
        d = self.dims
        inv_freq = 1.0 / (d.rope_theta ** (torch.arange(0, d.head_dim, 2, dtype=torch.int64).float() / d.head_dim))
        freqs = torch.outer(torch.arange(d.n_positions, dtype=torch.float32), inv_freq)
        for name, t in (("engine.rope_cos", freqs.cos()), ("engine.rope_sin", freqs.sin())):
            t = t.to(torch.bfloat16).contiguous()
            shape = (C.c_int64 * 2)(*t.shape)
            self._ck(self._lib.sv_engine_load_weight(self._h, name.encode(), C.c_void_p(t.data_ptr()), shape, 2,
                                                     _lib.SV_DTYPE_BF16))

    # -- stages --------------------------------------------------------------------------
    def _dev(self, t: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
        return t.to(device=self.device, dtype=dtype, non_blocking=True).contiguous()

    def encode_images(self, pixels: torch.Tensor, return_embeds: bool = False, return_vit: bool = False):
        """ViT + adapter. pixels [B,3,S,S] (any float dtype/device) -> resident visual prefix."""
        d = self.dims
        if pixels.dim() != 4 or tuple(pixels.shape[1:]) != (3, d.image_size, d.image_size):
            raise ValueError(f"image batch must be [B,3,{d.image_size},{d.image_size}], got {tuple(pixels.shape)}")
        px = self._dev(pixels, torch.bfloat16)
        B = px.shape[0]
        emb = torch.empty(B, d.query_length, d.hidden, dtype=torch.bfloat16, device=self.device) if return_embeds else None
        vit = torch.empty(B, d.query_length, d.vit_width, dtype=torch.bfloat16, device=self.device) if return_vit else None
        with self._lock:
            self._ck(self._lib.sv_encode_images(
                self._h, C.c_void_p(px.data_ptr()), B, C.c_void_p(emb.data_ptr() if emb is not None else 0),
                C.c_void_p(vit.data_ptr() if vit is not None else 0), _stream_ptr(self.device)))
            self._batch = B
        return emb, vit

    def prefill(self, prompt_ids: torch.Tensor, return_logits: bool = False) -> Optional[torch.Tensor]:
        ids = self._dev(prompt_ids, torch.int32)
        if ids.dim() != 2:
            raise ValueError("prompt_ids must be [B,P]")
        B, P = ids.shape
        logits = torch.empty(B, self.dims.vocab, dtype=torch.float32, device=self.device) if return_logits else None
        with self._lock:
            self._ck(self._lib.sv_prefill(self._h, C.c_void_p(ids.data_ptr()), B, P,
                                          C.c_void_p(logits.data_ptr() if logits is not None else 0),
                                          _stream_ptr(self.device)))
            self._prompt_len = P
            self._prefix_len = self.query_length + P
        return logits

    def prefill_embeds(self, inputs_embeds: torch.Tensor, return_logits: bool = False) -> Optional[torch.Tensor]:
        x = self._dev(inputs_embeds, torch.bfloat16)
        if x.dim() != 3 or x.shape[2] != self.dims.hidden:
            raise ValueError("inputs_embeds must be [B,T,hidden]")
        B, T, _ = x.shape
        logits = torch.empty(B, self.dims.vocab, dtype=torch.float32, device=self.device) if return_logits else None
        with self._lock:
            self._ck(self._lib.sv_prefill_embeds(self._h, C.c_void_p(x.data_ptr()), B, T,
                                                 C.c_void_p(logits.data_ptr() if logits is not None else 0),
                                                 _stream_ptr(self.device)))
            self._batch = B
            self._prefix_len = T
        return logits

    def decode_step(self, ids: torch.Tensor, return_logits: bool = True) -> Optional[torch.Tensor]:
        t = self._dev(ids, torch.int32).reshape(-1)
        if t.numel() != self._batch:
            raise ValueError("ids must have one entry per image of the current batch")
        logits = torch.empty(self._batch, self.dims.vocab, dtype=torch.float32, device=self.device) if return_logits else None
        with self._lock:
            self._ck(self._lib.sv_decode_step(self._h, C.c_void_p(t.data_ptr()),
                                              C.c_void_p(logits.data_ptr() if logits is not None else 0),
                                              _stream_ptr(self.device)))
        return logits

    def score(self, ids: torch.Tensor) -> torch.Tensor:
        """Teacher-forced log-likelihoods at prefill speed (`sv_score_tokens`): ids `[B, T]` are appended to the cache of the
        current batch and fp32 `[B, T]` is returned, `out[b, t] = log p(ids[b, t] | cache, ids[b, :t])` (t = 0 from the
        resident logits of the previous prefill / decode step / score call).  The tokens extend the prefix, so `decode_step`,
        `score` or `generate` may follow."""
        t = self._dev(ids, torch.int32)
        if t.dim() != 2 or t.shape[0] != self._batch:
            raise ValueError(f"ids must be [B, T] with B = the current batch ({self._batch}), got {tuple(t.shape)}")
        out = torch.empty(t.shape[0], t.shape[1], dtype=torch.float32, device=self.device)
        with self._lock:
            self._ck(self._lib.sv_score_tokens(self._h, C.c_void_p(t.data_ptr()), t.shape[0], t.shape[1],
                                               C.c_void_p(out.data_ptr()), _stream_ptr(self.device)))
        return out

    def reorder_cache(self, src_rows: torch.Tensor) -> None:
        """KV-cache row permutation for beam search: row r <- row src_rows[r]."""
        idx = self._dev(src_rows, torch.int32).reshape(-1)
        if idx.numel() != self._batch:
            raise ValueError("src_rows must have one entry per cache row")
        with self._lock:
            self._ck(self._lib.sv_reorder_cache(self._h, C.c_void_p(idx.data_ptr()), _stream_ptr(self.device)))

    def beam_search_device(self, batch: int, *, num_beams: int, max_new_tokens: int, do_sample: bool = False,
                           temperature: float = 1.0, top_p: float = 1.0, repetition_penalty: float = 1.0,
                           length_penalty: float = 1.0, early_stopping=True, eos_token_id: Optional[int] = 0,
                           pad_token_id: int = 0, stop_ids: Sequence[int] = (), seed: int = 0,
                           poll_interval: int = 16) -> torch.Tensor:
        """`sv_beam_search`: the whole beam search / beam-sample on the device, after a prefill of batch * num_beams rows
        (every image repeated num_beams times, adjacent).  Returns int32 `[batch, n_generated]`, the best hypothesis per image.
        Raises NotImplementedError when the vocabulary does not fit the candidate kernel (use the host-stepped loop)."""
        bp = BeamSearchParams(num_beams, max_new_tokens, do_sample, temperature, top_p, repetition_penalty, length_penalty,
                              early_stopping, eos_token_id, pad_token_id, stop_ids, seed, poll_interval).to_c()
        out = torch.empty(batch, max(int(max_new_tokens), 1), dtype=torch.int32, device=self.device)
        olen = torch.empty(batch, dtype=torch.int32, device=self.device)
        with self._lock:
            self._ck(self._lib.sv_beam_search(self._h, C.byref(bp), int(batch), C.c_void_p(out.data_ptr()),
                                              C.c_void_p(olen.data_ptr()), _stream_ptr(self.device)))
        return out[:, : int(olen[0].item())]

    def expand_batch(self, src_rows) -> None:
        """Prefix-KV sharing: right after a prefill, row r of the new batch becomes a copy of prefilled row src_rows[r]."""
        rows = [int(r) for r in src_rows]
        arr = (C.c_int32 * len(rows))(*rows)
        with self._lock:
            self._ck(self._lib.sv_expand_batch(self._h, arr, len(rows), _stream_ptr(self.device)))
        self._batch = len(rows)

    def generate(self, params: GenerationParams, on_tokens=None) -> torch.Tensor:
        """Run the decode loop after a prefill. Returns int32 [B, n_generated] (new tokens only).

        `on_tokens(ids, first_step)` (optional) streams: it is called on this thread every `params.poll_interval` steps and
        once at the end with a CPU int32 tensor `[B, n]` of the tokens generated since the previous call (`sv_generate_stream`);
        returning a truthy value cancels the generation.  An exception raised by the callback cancels and is re-raised."""
        B, n = self._batch, int(params.max_new_tokens)
        out = torch.empty(B, max(n, 1), dtype=torch.int32, device=self.device)
        olen = torch.empty(B, dtype=torch.int32, device=self.device)
        cp = params.to_c()
        spec = None
        if params.prompt_lookup_num_tokens > 0:        # one image: `sv_generate_speculative`, the same tokens as below
            spec = _lib.SpecParams(int(params.prompt_lookup_num_tokens), int(params.max_matching_ngram_size))
        if spec is not None and on_tokens is None:
            with self._lock:
                self._ck(self._lib.sv_generate_speculative(self._h, C.byref(cp), C.byref(spec), C.c_void_p(out.data_ptr()),
                                                           C.c_void_p(olen.data_ptr()), _lib.TOKEN_CALLBACK(), None,
                                                           _stream_ptr(self.device)))
        elif on_tokens is None:
            with self._lock:
                self._ck(self._lib.sv_generate(self._h, C.byref(cp), C.c_void_p(out.data_ptr()), C.c_void_p(olen.data_ptr()),
                                               _stream_ptr(self.device)))
        else:
            failure = []

            def trampoline(_user, ids_ptr, batch, first_step, n_steps):
                try:
                    flat = torch.frombuffer(C.cast(ids_ptr, C.POINTER(C.c_int32 * (batch * n_steps))).contents, dtype=torch.int32)
                    return 1 if on_tokens(flat.view(batch, n_steps).clone(), int(first_step)) else 0
                except BaseException as exc:      # never let an exception unwind through the C frames
                    failure.append(exc)
                    return 1

            cb = _lib.TOKEN_CALLBACK(trampoline)
            with self._lock:
                if spec is not None:
                    self._ck(self._lib.sv_generate_speculative(self._h, C.byref(cp), C.byref(spec), C.c_void_p(out.data_ptr()),
                                                               C.c_void_p(olen.data_ptr()), cb, None, _stream_ptr(self.device)))
                else:
                    self._ck(self._lib.sv_generate_stream(self._h, C.byref(cp), C.c_void_p(out.data_ptr()),
                                                          C.c_void_p(olen.data_ptr()), cb, None, _stream_ptr(self.device)))
            if failure:
                raise failure[0]
        n_gen = int(olen[0].item())
        return out[:, :n_gen]

    def spec_verify_step(self, ids) -> torch.Tensor:
        """Teacher-forced verify forward (`sv_spec_verify_step`) after a one-image prefill: the logits, fp32 `[len(ids),
        vocab]`, of ids fed as the columns of one speculative verify step at the next positions (the cache does not advance)."""
        ids = [int(t) for t in ids]
        logits = torch.empty(len(ids), self.dims.vocab, dtype=torch.float32, device=self.device)
        with self._lock:
            self._ck(self._lib.sv_spec_verify_step(self._h, (C.c_int32 * len(ids))(*ids), len(ids),
                                                   C.c_void_p(logits.data_ptr()), _stream_ptr(self.device)))
        return logits

    def last_spec_stats(self) -> Dict[str, int]:
        """Counters of the last speculative `generate` (`sv_last_spec_stats`): verify steps, drafts proposed, drafts accepted."""
        v = [C.c_int32() for _ in range(3)]
        self._ck(self._lib.sv_last_spec_stats(self._h, *(C.byref(x) for x in v)))
        return {"steps": v[0].value, "drafted": v[1].value, "accepted": v[2].value}

    def generate_im2svg_host(self, pixels_host: torch.Tensor, prompt_ids_host: torch.Tensor,
                             params: GenerationParams) -> Tuple[torch.Tensor, int]:
        """Whole path on HOST buffers (pinned CPU tensors in, CPU tensors out): the e2e entry point."""
        d = self.dims
        if pixels_host.is_cuda or prompt_ids_host.is_cuda:
            raise ValueError("host entry point takes CPU tensors")
        px = pixels_host.to(torch.bfloat16).contiguous()
        ids = prompt_ids_host.to(torch.int32).contiguous()
        B, P = ids.shape
        out = torch.empty(B, int(params.max_new_tokens), dtype=torch.int32).pin_memory()
        olen = torch.empty(B, dtype=torch.int32).pin_memory()
        cp = params.to_c()
        with self._lock:
            self._ck(self._lib.sv_generate_im2svg_host(
                self._h, C.c_void_p(px.data_ptr()), B, C.c_void_p(ids.data_ptr()), P, C.byref(cp),
                C.c_void_p(out.data_ptr()), C.c_void_p(olen.data_ptr()), _stream_ptr(self.device)))
            self._batch = B
        n_gen = int(olen[0])
        return out[:, :n_gen], n_gen

    # -- continuous batching (sv_session_*) -----------------------------------------------------
    def generate_requests(self, pixels: torch.Tensor, prompt_ids: torch.Tensor, params: GenerationParams, *,
                          max_new_tokens: Optional[Sequence[int]] = None, seeds: Optional[Sequence[int]] = None, n: int = 1,
                          on_finish=None, slots: Optional[int] = None) -> List[torch.Tensor]:
        """Continuous batching over any number of images: a decode session of `slots` (default `max_batch`) cache rows,
        refilled with the next queued image whenever a row finishes (`ContinuousScheduler`).  Completion j of image i
        (index i * n + j of the returned list, int32 on the CPU) holds exactly the tokens a one-image `generate` of image i
        with `params` (seed `seeds[i * n + j]`, default `params.seed + i * n + j`, and `max_new_tokens[i]` new tokens at most)
        returns.  `params.max_new_tokens` is the session cap; `on_finish(index, ids)` streams results as they complete.
        `params.prompt_lookup_num_tokens > 0` asks for a speculative session (see `session_begin`): same tokens."""
        from .continuous import ContinuousScheduler

        return ContinuousScheduler(self, slots).run(pixels, prompt_ids, params, max_new_tokens=max_new_tokens, seeds=seeds,
                                                    n=n, on_finish=on_finish)

    @property
    def fused_decode(self) -> bool:
        """The engine decodes through the fused graph path (not `SV_DECODE=legacy`)."""
        return "decode=legacy-kernels" not in self.describe()

    def session_begin(self, params: GenerationParams, slots: int) -> None:
        """Open a decode session of `slots` cache rows.  `params.prompt_lookup_num_tokens` / `max_matching_ngram_size` are a
        speed hint: on v1 engines on the fused decode path with `slots >= 2`, the session drafts up to that many tokens
        (clamped to `slots - 1`) per row into the columns idle slots leave (`sv_session_begin_speculative`); otherwise it
        runs plain.  Either way every request gets the same tokens."""
        from .continuous import spec_session_k

        cp = params.to_c()
        k = spec_session_k(params, slots, self)
        with self._lock:
            if k > 0:
                sp = _lib.SpecParams(k, int(params.max_matching_ngram_size))
                self._ck(self._lib.sv_session_begin_speculative(self._h, C.byref(cp), C.byref(sp), int(slots)))
            else:
                self._ck(self._lib.sv_session_begin(self._h, C.byref(cp), int(slots)))
            self._session_slots = int(slots)
            self._session_spec = k > 0
            self._batch = 0

    def session_spec_stats(self) -> Optional[Dict[str, int]]:
        """Counters of the open speculative session (`sv_session_spec_stats`): verify steps, drafts proposed, drafts
        accepted; None when the open session is a plain one."""
        if not getattr(self, "_session_spec", False):
            return None
        v = [C.c_int32() for _ in range(3)]
        with self._lock:
            self._ck(self._lib.sv_session_spec_stats(self._h, *(C.byref(x) for x in v)))
        return {"steps": v[0].value, "drafted": v[1].value, "accepted": v[2].value}

    def session_admit(self, pixels: torch.Tensor, prompt_ids: torch.Tensor, slots: Sequence[int], *,
                      max_new_tokens: Optional[Sequence[int]] = None, seeds: Optional[Sequence[int]] = None,
                      src: Optional[Sequence[int]] = None) -> None:
        """Encode and prefill images `[n_img, 3, S, S]` (prompts `[n_img, P]`) into free `slots`; `src[j]` is the image of
        slots[j] (default j), so one image may fill several slots (n completions, prefilled once)."""
        d = self.dims
        if pixels.dim() != 4 or tuple(pixels.shape[1:]) != (3, d.image_size, d.image_size):
            raise ValueError(f"image batch must be [B,3,{d.image_size},{d.image_size}], got {tuple(pixels.shape)}")
        px = self._dev(pixels, torch.bfloat16)
        ids = self._dev(prompt_ids, torch.int32)
        k = len(slots)
        def arr(t, v, mask=None):
            return None if v is None else (t * k)(*[int(x) & mask if mask else int(x) for x in v])

        sl, mx, sr = arr(C.c_int32, slots), arr(C.c_int32, max_new_tokens), arr(C.c_int32, src)
        sd = arr(C.c_uint64, seeds, 2 ** 64 - 1)
        with self._lock:
            self._ck(self._lib.sv_session_admit(self._h, C.c_void_p(px.data_ptr()), k, C.c_void_p(ids.data_ptr()), ids.shape[1],
                                                sl, mx, sd, sr, _stream_ptr(self.device)))

    def session_run(self, max_steps: int) -> Tuple[int, List[bool], List[int]]:
        """Replay decode steps until a slot finishes: (steps run, finished flag per slot, tokens per slot)."""
        S = self._session_slots
        fin, ln = (C.c_int32 * S)(), (C.c_int32 * S)()
        with self._lock:
            r = self._lib.sv_session_run(self._h, int(max_steps), fin, ln, _stream_ptr(self.device))
            if r < 0:
                self._ck(r)
        return int(r), [bool(v) for v in fin], [int(v) for v in ln]

    def session_read(self, slot: int) -> torch.Tensor:
        """The tokens of `slot` as of the last `session_run` (int32, CPU)."""
        out = torch.empty(self.dims.max_len, dtype=torch.int32)
        with self._lock:
            r = self._lib.sv_session_read(self._h, int(slot), C.c_void_p(out.data_ptr()), _stream_ptr(self.device))
            if r < 0:
                self._ck(r)
        return out[:r].clone()

    def beam_requests(self, pixels: torch.Tensor, prompt_ids: torch.Tensor, *, num_beams: int, max_new_tokens: int,
                      caps: Optional[Sequence[int]] = None, seeds: Optional[Sequence[int]] = None, do_sample: bool = False,
                      temperature: float = 1.0, top_p: float = 1.0, repetition_penalty: float = 1.0,
                      length_penalty: float = 1.0, early_stopping=True, eos_token_id: Optional[int] = 0, pad_token_id: int = 0,
                      stop_ids: Sequence[int] = (), seed: int = 0, poll_interval: int = 16, on_finish=None,
                      slots: Optional[int] = None) -> List[torch.Tensor]:
        """Continuous batching of beam search over any number of images: a beam session of `slots` cache rows (default
        `max_batch` rounded down to a multiple of `num_beams`) in groups of `num_beams`, each group refilled with the next
        queued image as soon as its search ends.  Image k gets the int32 ids (CPU) that
        `beam_search(engine, pixels[k:k+1], prompt, num_beams=..., impl="device", seed=seeds[k], max_new_tokens=caps[k], ...)`
        returns, bit for bit, when its cap is the session cap `max_new_tokens` (a smaller cap: when the decode attention's
        partition of prefix + cap is that of prefix + max_new_tokens).  `seeds` default to `seed + k`; `on_finish(k, ids)`
        streams results as they complete."""
        from .continuous import ContinuousScheduler

        fill = (pad_token_id if pad_token_id is not None else eos_token_id) if eos_token_id is not None else -1
        params = BeamSearchParams(num_beams, max_new_tokens, do_sample, temperature, top_p, repetition_penalty, length_penalty,
                                  early_stopping, eos_token_id, fill, stop_ids, seed, poll_interval)
        if slots is None:
            slots = self.dims.max_batch // int(num_beams) * int(num_beams)
        return ContinuousScheduler(self, slots, num_beams=num_beams).run(pixels, prompt_ids, params, max_new_tokens=caps,
                                                                         seeds=seeds, on_finish=on_finish)

    def beam_session_begin(self, params: BeamSearchParams, slots: int) -> None:
        bp = params.to_c()
        with self._lock:
            self._ck(self._lib.sv_beam_session_begin(self._h, C.byref(bp), int(slots)))
            self._session_slots = int(slots)
            self._session_spec = False
            self._batch = 0

    def beam_session_admit(self, pixels: torch.Tensor, prompt_ids: torch.Tensor, groups: Sequence[int], *,
                           max_new_tokens: Optional[Sequence[int]] = None, seeds: Optional[Sequence[int]] = None) -> None:
        """Encode and prefill images `[k, 3, S, S]` (prompts `[k, P]`) into the free beam groups `groups` (group g = slots
        g * num_beams ...); image j runs its own search with cap `max_new_tokens[j]` and seed `seeds[j]`."""
        d = self.dims
        if pixels.dim() != 4 or tuple(pixels.shape[1:]) != (3, d.image_size, d.image_size):
            raise ValueError(f"image batch must be [B,3,{d.image_size},{d.image_size}], got {tuple(pixels.shape)}")
        px = self._dev(pixels, torch.bfloat16)
        ids = self._dev(prompt_ids, torch.int32)
        k = len(groups)
        if px.shape[0] != k or ids.dim() != 2 or ids.shape[0] != k:
            raise ValueError(f"{k} groups need {k} images and [{k}, P] prompt ids")
        gr = (C.c_int32 * k)(*[int(g) for g in groups])
        mx = None if max_new_tokens is None else (C.c_int32 * k)(*[int(m) for m in max_new_tokens])
        sd = None if seeds is None else (C.c_uint64 * k)(*[int(x) & (2 ** 64 - 1) for x in seeds])
        with self._lock:
            self._ck(self._lib.sv_beam_session_admit(self._h, C.c_void_p(px.data_ptr()), k, C.c_void_p(ids.data_ptr()),
                                                     ids.shape[1], gr, mx, sd, _stream_ptr(self.device)))

    def session_end(self) -> None:
        with self._lock:
            self._ck(self._lib.sv_session_end(self._h))
            self._session_spec = False

    # -- introspection -------------------------------------------------------------------
    def launch_count(self) -> int:
        return int(self._lib.sv_launch_count(self._h))

    def describe(self) -> str:
        return self._lib.sv_engine_describe(self._h).decode()

    def debug_timeline(self, n: int = 1024, raw: bool = False):
        buf = (C.c_longlong * n)()
        self._ck(self._lib.sv_debug_read_timeline(self._h, buf, n))
        return [int(v) for v in buf] if raw else [int(v) for v in buf if v]

    def last_decode_timing(self) -> Tuple[float, int]:
        ms, steps = C.c_float(), C.c_int32()
        self._ck(self._lib.sv_last_decode_timing(self._h, C.byref(ms), C.byref(steps)))
        return float(ms.value), int(steps.value)


# -- single-kernel entry points (unit parity tests) --------------------------------------------
def _p(t: Optional[torch.Tensor]) -> C.c_void_p:
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def op_layernorm(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    lib = _lib.load()
    y = torch.empty_like(x)
    rows = x.numel() // x.shape[-1]
    _lib.check(lib, lib.sv_op_layernorm(_p(x), _p(w), _p(b), _p(y), rows, x.shape[-1], eps, _stream_ptr(x.device)))
    return y


def op_linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None,
              residual: Optional[torch.Tensor] = None, act: int = 0, impl: int = 0) -> torch.Tensor:
    lib = _lib.load()
    M, K = x.shape
    N = w.shape[0]
    y = torch.empty(M, N, dtype=torch.bfloat16, device=x.device)
    _lib.check(lib, lib.sv_op_linear(impl, _p(x), _p(w), _p(bias), _p(residual), _p(y), M, N, K, act, _stream_ptr(x.device)))
    return y


def op_attention_vit(qkv: torch.Tensor, batch: int, seq: int, heads: int) -> torch.Tensor:
    lib = _lib.load()
    out = torch.empty(batch * seq, heads * 64, dtype=torch.bfloat16, device=qkv.device)
    _lib.check(lib, lib.sv_op_attention_vit(_p(qkv), _p(out), batch, seq, heads, _stream_ptr(qkv.device)))
    return out


def op_attention_mqa(qkv: torch.Tensor, batch: int, seq: int, heads: int) -> torch.Tensor:
    lib = _lib.load()
    out = torch.empty(batch * seq, heads * 128, dtype=torch.bfloat16, device=qkv.device)
    _lib.check(lib, lib.sv_op_attention_mqa(_p(qkv), _p(out), batch, seq, heads, _stream_ptr(qkv.device)))
    return out


def op_attention_chunk(qkv: torch.Tensor, batch: int, seq: int, q0: int, n_head: int, n_kv: int, window: int = 0) -> torch.Tensor:
    """Queries of positions [q0, seq) against a cache of all `seq` positions of packed qkv `[batch * seq, (n_head + 2 n_kv) * 128]`."""
    lib = _lib.load()
    out = torch.empty(batch * (seq - q0), n_head * 128, dtype=torch.bfloat16, device=qkv.device)
    _lib.check(lib, lib.sv_op_attention_chunk(_p(qkv), _p(out), batch, seq, q0, n_head, n_kv, window, _stream_ptr(qkv.device)))
    return out


def op_lm_logprob(x: torch.Tensor, w: torch.Tensor, targets: torch.Tensor) -> torch.Tensor:
    """`log_softmax(float(bf16(x @ w.T)))[m, targets[m]]`, fp32 `[M]`, without materialising the logits."""
    lib = _lib.load()
    M, K = x.shape
    tg = targets.to(device=x.device, dtype=torch.int32).contiguous()
    out = torch.empty(M, dtype=torch.float32, device=x.device)
    _lib.check(lib, lib.sv_op_lm_logprob(_p(x), _p(w), _p(tg), _p(out), M, w.shape[0], K, _stream_ptr(x.device)))
    return out


def op_im2col(pixels: torch.Tensor, patch: int, kpad: int) -> torch.Tensor:
    """bf16 `pixels [B, 3, S, S]` -> patches `[B * (S / patch)^2, kpad]` (columns (c, iy, ix), zero-padded to kpad)."""
    lib = _lib.load()
    B, S = pixels.shape[0], pixels.shape[-1]
    out = torch.empty(B * (S // patch) ** 2, kpad, dtype=torch.bfloat16, device=pixels.device)
    _lib.check(lib, lib.sv_op_im2col(_p(pixels), _p(out), B, S, patch, kpad, _stream_ptr(pixels.device)))
    return out


def op_vit_assemble(pe: torch.Tensor, cls: Optional[torch.Tensor], pos: torch.Tensor, batch: int) -> torch.Tensor:
    """`bf16(cat(cls, pe) + pos)` per image (`pe [batch * np, width]`), or `bf16(pe + pos)` without cls."""
    lib = _lib.load()
    width = pe.shape[-1]
    np_ = pe.numel() // width // batch
    q = np_ + (cls is not None)
    x = torch.empty(batch * q, width, dtype=torch.bfloat16, device=pe.device)
    _lib.check(lib, lib.sv_op_vit_assemble(_p(pe), _p(cls), _p(pos), _p(x), batch, np_, width, _stream_ptr(pe.device)))
    return x


def op_adapter_norm(kind: int, z: torch.Tensor, w: torch.Tensor, b: torch.Tensor, rmean: Optional[torch.Tensor] = None,
                    rvar: Optional[torch.Tensor] = None, eps: float = 1e-5) -> torch.Tensor:
    """The adapter norm over `z [B, Q, H]`: LayerNorm([Q, H]) (`kind` SV_ADAPTER_NORM_SLAB, w / b `[Q, H]`) or eval
    BatchNorm1d(Q) (SV_ADAPTER_NORM_TOKENS, w / b / rmean / rvar `[Q]`)."""
    lib = _lib.load()
    B, Q, H = z.shape
    y = torch.empty_like(z)
    _lib.check(lib, lib.sv_op_adapter_norm(kind, _p(z), _p(w), _p(b), _p(rmean), _p(rvar), _p(y), B, Q, H, eps,
                                           _stream_ptr(z.device)))
    return y


def op_embed_prefix(visual: Optional[torch.Tensor], ids: Optional[torch.Tensor], wte: torch.Tensor, wpe: Optional[torch.Tensor],
                    batch: int, q: int, p: int, pos0: int = 0, id_stride: Optional[int] = None) -> torch.Tensor:
    """`[batch * (q + p), h]`: visual rows then `wte[clamp(id)]` rows, `+ wpe[pos0 + t]` unless wpe is None.  `ids` int32
    with row b's ids at `b * id_stride` (default p)."""
    lib = _lib.load()
    h, vocab = wte.shape[1], wte.shape[0]
    x = torch.empty(batch * (q + p), h, dtype=torch.bfloat16, device=wte.device)
    _lib.check(lib, lib.sv_op_embed_prefix(_p(visual), _p(ids), _p(wte), _p(wpe), _p(x), batch, q, p, h, vocab, pos0,
                                           p if id_stride is None else id_stride, _stream_ptr(wte.device)))
    return x


def op_attention_prefill(qkv: torch.Tensor, kcache: torch.Tensor, vtcache: torch.Tensor, seq: int, n_head: int, n_kv: int,
                         window: int = 0) -> torch.Tensor:
    """The prefill attention over caller-owned caches `kcache [>= B, n_kv, tcap, 128]`, `vtcache [>= B, n_kv, 128, tcap]`:
    slots `[0, seq)` of images `b < B` get the K/V of packed qkv `[B * seq, (n_head + 2 n_kv) * 128]`, then causal attention
    -> `[B * seq, n_head * 128]`."""
    lib = _lib.load()
    B, tcap = qkv.shape[0] // seq, kcache.shape[2]
    out = torch.empty(B * seq, n_head * 128, dtype=torch.bfloat16, device=qkv.device)
    _lib.check(lib, lib.sv_op_attention_prefill(_p(qkv), _p(kcache), _p(vtcache), _p(out), B, seq, n_head, n_kv, tcap, window,
                                                _stream_ptr(qkv.device)))
    return out


def op_lm_logits(x: torch.Tensor, w: torch.Tensor, y: Optional[torch.Tensor] = None) -> torch.Tensor:
    """`bf16(x @ w.T)` for any N on the scoring lm_head tiling; `y` (at least M * N elements) may be given."""
    lib = _lib.load()
    M, K = x.shape
    N = w.shape[0]
    if y is None:
        y = torch.empty(M, N, dtype=torch.bfloat16, device=x.device)
    _lib.check(lib, lib.sv_op_lm_logits(_p(x), _p(w), _p(y), M, N, K, _stream_ptr(x.device)))
    return y


def op_attention_score(qkv: torch.Tensor, kcache: torch.Tensor, vtcache: torch.Tensor, chunk: int, pos0: int, n_head: int,
                       n_kv: int, window: int = 0) -> torch.Tensor:
    """The scoring chunk attention over caller-owned caches `kcache [>= B, n_kv, tcap, 128]`, `vtcache [>= B, n_kv, 128,
    tcap]`: row `[b][t]` of packed qkv `[B * chunk, (n_head + 2 n_kv) * 128]` is position `pos0 + t`; its K/V go to slot
    `pos0 + t` of image b, then it attends causally to slots `[0, pos0 + t]` -> `[B * chunk, n_head * 128]`."""
    lib = _lib.load()
    B, tcap = qkv.shape[0] // chunk, kcache.shape[2]
    out = torch.empty(B * chunk, n_head * 128, dtype=torch.bfloat16, device=qkv.device)
    _lib.check(lib, lib.sv_op_attention_score(_p(qkv), _p(kcache), _p(vtcache), _p(out), B, chunk, pos0, n_head, n_kv, tcap,
                                              window, _stream_ptr(qkv.device)))
    return out


def op_logits_logprob(logits: torch.Tensor, targets: torch.Tensor) -> torch.Tensor:
    """`log_softmax(float(logits))[m, targets[m]]` over bf16 `logits [M, vocab]`, fp32 `[M]` (NaN where a target lies
    outside [0, vocab)): position 0 of a scoring call."""
    lib = _lib.load()
    M, V = logits.shape
    tg = targets.to(device=logits.device, dtype=torch.int32).contiguous()
    out = torch.empty(M, dtype=torch.float32, device=logits.device)
    _lib.check(lib, lib.sv_op_logits_logprob(_p(logits), _p(tg), _p(out), M, V, _stream_ptr(logits.device)))
    return out


def _i32s(v) -> C.Array:
    v = [int(a) for a in v]
    return (C.c_int32 * max(1, len(v)))(*v)


def op_attention_decode(qkv: torch.Tensor, kcache: torch.Tensor, vtcache: torch.Tensor, lens, n_head: int, n_kv: int,
                        nsplit: int, window: int = 0, impl: int = _lib.SV_ATTN_DECODE_SPLIT, per_row: int = 0) -> torch.Tensor:
    """One decode-attention launch over caller-filled caches `kcache [B, n_kv, tcap, 128]`, `vtcache [B, n_kv, 128, tcap]`:
    row b's query (qkv row b) attends to keys `[0, lens[b])` -> `[B, n_head * 128]`.  `per_row=2` (cluster only): the column
    map of a verify step, qkv row c attends to keys `[0, lens[c]]` of cache row 0, `B` = qkv's rows."""
    lib = _lib.load()
    B, tcap = (qkv.shape[0] if int(per_row) == 2 else kcache.shape[0]), kcache.shape[2]
    out = torch.empty(B, n_head * 128, dtype=torch.bfloat16, device=qkv.device)
    _lib.check(lib, lib.sv_op_attention_decode(impl, int(per_row), _p(qkv), _p(kcache), _p(vtcache), _p(out), _i32s(lens), B,
                                               n_head, n_kv, tcap, nsplit, window, _stream_ptr(qkv.device)))
    return out


def op_gemv_ring(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
                 ln: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, act: int = 0, epi: int = 0, tiled: bool = False,
                 ln_eps: float = 1e-5, y: Optional[torch.Tensor] = None, kcache: Optional[torch.Tensor] = None,
                 vtcache: Optional[torch.Tensor] = None, n_head: int = 0, n_kv: int = 0, pos=None, per_row: int = 0,
                 n_live: int = 0):
    """One weight-ring GEMV launch (the decode step's): `y [B, N]`; with `epi=2` also the argmax partials
    `(amax_val, amax_idx)`, `[ntiles, row_stride]`.  `y` may be `residual` (in place).  `epi=1, per_row=2`: the column map of
    a verify step, column c's K/V appended in cache row 0 at `pos[c]` for `c < n_live` (passed as `pos_host[B]`)."""
    lib = _lib.load()
    B, K = x.shape
    N = w.shape[0]
    if y is None:
        y = torch.empty(B, N, dtype=torch.bfloat16, device=x.device)
    a = _lib.OpRing(x=x.data_ptr(), w=w.data_ptr(), y=y.data_ptr(), B=B, N=N, K=K, act=act, epi=epi, tiled=int(tiled),
                    ln_eps=ln_eps, n_head=n_head, n_kv=n_kv, per_row=int(per_row))
    if bias is not None:
        a.bias = bias.data_ptr()
    if residual is not None:
        a.residual = residual.data_ptr()
    if ln is not None:
        a.ln_w, a.ln_b = ln[0].data_ptr(), ln[1].data_ptr()
    if kcache is not None:
        a.kcache, a.vtcache, a.tcap = kcache.data_ptr(), vtcache.data_ptr(), kcache.shape[2]
    if pos is not None:
        posv = _i32s(list(pos) + ([n_live] if int(per_row) == 2 else []))
        a.pos_host = C.cast(posv, C.POINTER(C.c_int32))
    amax = None
    if epi == 2:
        nt, rs = lib.sv_op_ring_ntiles(N), lib.sv_op_ring_row_stride(B)
        amax = (torch.full((nt, rs), float("nan"), dtype=torch.float32, device=x.device),
                torch.full((nt, rs), -1, dtype=torch.int32, device=x.device))
        a.amax_val, a.amax_idx = amax[0].data_ptr(), amax[1].data_ptr()
    _lib.check(lib, lib.sv_op_gemv_ring(C.byref(a), _stream_ptr(x.device)))
    return (y, amax) if epi == 2 else y


def op_rope_table(max_pos: int, d: int, theta: float, device="cuda") -> Tuple[torch.Tensor, torch.Tensor]:
    """The engine's bf16 RoPE tables `cos, sin [max_pos, d / 2]`."""
    lib = _lib.load()
    cos = torch.empty(max_pos, d // 2, dtype=torch.bfloat16, device=device)
    sin = torch.empty_like(cos)
    _lib.check(lib, lib.sv_op_rope_table(_p(cos), _p(sin), max_pos, d, theta, _stream_ptr(cos.device)))
    return cos, sin


def op_rope(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, n_head: int, n_kv: int, seq: int = 1, pos0: int = 0,
            pos=None, per_row: bool = False, kcache: Optional[torch.Tensor] = None,
            vtcache: Optional[torch.Tensor] = None) -> torch.Tensor:
    """RoPE in place on packed qkv rows `[rows, (n_head + 2 n_kv) * 128]` (see sv_op_rope); returns qkv."""
    lib = _lib.load()
    tcap = kcache.shape[2] if kcache is not None else 0
    posv = _i32s(pos) if pos is not None else None
    _lib.check(lib, lib.sv_op_rope(_p(qkv), _p(cos), _p(sin), qkv.shape[0], seq, n_head, n_kv, cos.shape[0], pos0, posv,
                                   int(per_row), _p(kcache), _p(vtcache), tcap, _stream_ptr(qkv.device)))
    return qkv


def op_select(impl: int, logits: torch.Tensor, params: GenerationParams, seen: torch.Tensor, out_ids: torch.Tensor,
              next_ids: torch.Tensor, state: dict, per_row: bool = False, advance_len: int = 1, nsteps: int = 1,
              amax: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, wte: Optional[torch.Tensor] = None,
              wpe: Optional[torch.Tensor] = None, x: Optional[torch.Tensor] = None, n_positions: int = 0) -> dict:
    """`nsteps` token selections from bf16 `logits [B, vocab]` (see sv_op_select); `seen` uint8 `[B, vocab]`, `out_ids` int32
    `[B, out_stride]`, `next_ids` int32 `[B]` and (fused) `x` are updated in place.  `state` holds the generation state and
    is updated too: `step, cur_len, done, unfinished[B]`, or with `per_row` `row_len, row_step, row_active, row_max_new,
    row_seed` (`[B]` each), `row_mask, event`."""
    lib = _lib.load()
    B, vocab = logits.shape
    a = _lib.OpSelect(impl=impl, per_row=int(per_row), logits=logits.data_ptr(), vocab=vocab, B=B, params=params.to_c(),
                      seen=seen.data_ptr(), out_ids=out_ids.data_ptr(), next_ids=next_ids.data_ptr(),
                      out_stride=out_ids.shape[1], advance_len=advance_len, nsteps=nsteps)
    i32p = C.POINTER(C.c_int32)
    if per_row:
        keys = ("row_len", "row_step", "row_active", "row_max_new")
        arrs = {k: _i32s(state[k]) for k in keys}
        seeds = (C.c_uint64 * B)(*[int(s) & (2 ** 64 - 1) for s in state["row_seed"]])
        event = _i32s([state["event"]])
        for k in keys:
            setattr(a, k + "_host", C.cast(arrs[k], i32p))
        a.row_seed_host, a.event_host = C.cast(seeds, C.POINTER(C.c_uint64)), C.cast(event, i32p)
        a.row_mask = int(state["row_mask"])
    else:
        counters = _i32s([state["step"], state["cur_len"], state["done"]])
        unfinished = _i32s(state["unfinished"])
        a.counters_host, a.unfinished_host = C.cast(counters, i32p), C.cast(unfinished, i32p)
    if amax is not None:
        a.amax_val, a.amax_idx = amax[0].data_ptr(), amax[1].data_ptr()
    if wte is not None:
        a.wte, a.h = wte.data_ptr(), wte.shape[1]
    if wpe is not None:
        a.wpe = wpe.data_ptr()
    if x is not None:
        a.x = x.data_ptr()
    a.n_positions = n_positions
    _lib.check(lib, lib.sv_op_select(C.byref(a), _stream_ptr(logits.device)))
    if per_row:
        for k in keys:
            state[k] = list(arrs[k])[:B]
        state["row_seed"], state["event"] = list(seeds), int(event[0])
    else:
        state["step"], state["cur_len"], state["done"] = (int(v) for v in counters)
        state["unfinished"] = list(unfinished)[:B]
    return state


def op_spec_select(impl: int, params: GenerationParams, seen: torch.Tensor, out_ids: torch.Tensor, next_ids: torch.Tensor,
                   state: dict, spec: "_lib.SpecState", wte: torch.Tensor, wpe: Optional[torch.Tensor], x: torch.Tensor,
                   n_positions: int, logits: Optional[torch.Tensor] = None,
                   amax: Optional[Tuple[torch.Tensor, torch.Tensor]] = None) -> dict:
    """One speculative verify step's selection (see sv_op_spec_select) on one image row: bf16 `logits [ncols, vocab]`
    (GREEDY, SAMPLE); `seen` uint8 `[vocab]`, `out_ids` int32 `[out_stride]` (the history), `next_ids` int32 `[1]` and
    `x [ncols, h]` are updated in place, as are `spec` (a `_lib.SpecState`) and `state`: `step, cur_len, done, unfinished`."""
    lib = _lib.load()
    vocab = wte.shape[0]
    gen = _i32s([state["step"], state["cur_len"], state["done"], state["unfinished"]])
    a = _lib.OpSpec(impl=impl, vocab=vocab, params=params.to_c(), seen=seen.data_ptr(), out_ids=out_ids.data_ptr(),
                    next_ids=next_ids.data_ptr(), out_stride=out_ids.shape[-1], gen_host=C.cast(gen, C.POINTER(C.c_int32)),
                    spec_host=C.pointer(spec), wte=wte.data_ptr(), x=x.data_ptr(), h=wte.shape[1], n_positions=n_positions)
    if logits is not None:
        a.logits = logits.data_ptr()
    if wpe is not None:
        a.wpe = wpe.data_ptr()
    if amax is not None:
        a.amax_val, a.amax_idx = amax[0].data_ptr(), amax[1].data_ptr()
    _lib.check(lib, lib.sv_op_spec_select(C.byref(a), _stream_ptr(seen.device)))
    state["step"], state["cur_len"], state["done"], state["unfinished"] = (int(v) for v in gen)
    return state


def op_spec_session_select(impl: int, params: GenerationParams, seen: torch.Tensor, out_ids: torch.Tensor,
                           next_ids: torch.Tensor, rows: "_lib.SessionRows", ss: "_lib.SpecSessionState", wte: torch.Tensor,
                           wpe: Optional[torch.Tensor], x: torch.Tensor, n_positions: int, tcap: int,
                           logits: Optional[torch.Tensor] = None, amax: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
                           accept: bool = True) -> None:
    """One speculative-session kernel launch (see sv_op_spec_session_select) over S = ss.ncols slots: bf16 `logits [S,
    vocab]` (GREEDY, SAMPLE); `seen` uint8 `[S, vocab]`, `out_ids` int32 `[S, out_stride]`, `next_ids` int32 `[S]` and
    `x [S, h]` are updated in place, as are `rows` (a `_lib.SessionRows`) and `ss` (a `_lib.SpecSessionState`)."""
    lib = _lib.load()
    a = _lib.OpSpecSession(impl=impl, accept=int(bool(accept)), vocab=wte.shape[0], params=params.to_c(), seen=seen.data_ptr(),
                           out_ids=out_ids.data_ptr(), next_ids=next_ids.data_ptr(), out_stride=out_ids.shape[-1], tcap=tcap,
                           rows_host=C.pointer(rows), ss_host=C.pointer(ss), wte=wte.data_ptr(), x=x.data_ptr(),
                           h=wte.shape[1], n_positions=n_positions)
    if logits is not None:
        a.logits = logits.data_ptr()
    if wpe is not None:
        a.wpe = wpe.data_ptr()
    if amax is not None:
        a.amax_val, a.amax_idx = amax[0].data_ptr(), amax[1].data_ptr()
    _lib.check(lib, lib.sv_op_spec_session_select(C.byref(a), _stream_ptr(seen.device)))


def op_beam_candidates(logits: torch.Tensor, bp: "_lib.BeamParams", batch: int, cur_len: int, running_scores,
                       run_seq: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """One beam-candidates launch over bf16 `logits [batch * num_beams, vocab]` (see sv_op_beam_candidates); `run_seq` int32
    `[R, seq_stride]` holds each beam's generated ids -> `(cand_key, cand_val, cand_tok)`, `[R, 2 * num_beams]` each."""
    lib = _lib.load()
    R, vocab = logits.shape
    K = 2 * bp.num_beams
    key = torch.full((R, K), float("nan"), dtype=torch.float32, device=logits.device)
    val = torch.full_like(key, float("nan"))
    tok = torch.full((R, K), -1, dtype=torch.int32, device=logits.device)
    rs = (C.c_float * max(1, len(running_scores)))(*[float(v) for v in running_scores])
    _lib.check(lib, lib.sv_op_beam_candidates(_p(logits), vocab, C.byref(bp), batch, cur_len, rs, _p(run_seq), run_seq.shape[1],
                                              _p(key), _p(val), _p(tok), _stream_ptr(logits.device)))
    return key, val, tok


def op_beam_step(bp: "_lib.BeamParams", batch: int, vocab: int, state: "_lib.BeamState", cand, run_seq: torch.Tensor,
                 fin_seq: torch.Tensor, gen: list, advance: int, wte: torch.Tensor, wpe: Optional[torch.Tensor], x: torch.Tensor,
                 n_positions: int, next_ids: torch.Tensor, plan: "_lib.BeamPlan") -> None:
    """One beam-step launch (see sv_op_beam_step): `cand = (cand_key, cand_val, cand_tok)` `[R, 2 * num_beams]`; `run_seq`,
    `fin_seq` int32 `[2, R, seq_stride]`, `x [R, h]` and `next_ids` int32 `[R]` are updated in place, as are `state` (a
    `_lib.BeamState`), `plan` (a `_lib.BeamPlan`) and `gen = [cur_len, done]`."""
    lib = _lib.load()
    g = _i32s(gen)
    a = _lib.OpBeamStep(params=C.pointer(bp), batch=batch, vocab=vocab, seq_stride=run_seq.shape[-1], advance=advance,
                        state_host=C.pointer(state), cand_key=cand[0].data_ptr(), cand_val=cand[1].data_ptr(),
                        cand_tok=cand[2].data_ptr(), run_seq=run_seq.data_ptr(), fin_seq=fin_seq.data_ptr(),
                        gen_host=C.cast(g, C.POINTER(C.c_int32)), wte=wte.data_ptr(), x=x.data_ptr(), h=wte.shape[1],
                        n_positions=n_positions, next_ids=next_ids.data_ptr(), plan_host=C.pointer(plan))
    if wpe is not None:
        a.wpe = wpe.data_ptr()
    _lib.check(lib, lib.sv_op_beam_step(C.byref(a), _stream_ptr(x.device)))
    gen[:] = [int(g[0]), int(g[1])]


def op_beam_kv_copy(kcache: torch.Tensor, vtcache: torch.Tensor, rows: int, plan: "_lib.BeamPlan") -> None:
    """The KV suffix copies of a beam step (see sv_op_beam_kv_copy) in place over `kcache [n_layer, rows_cap, n_kv, tcap, 128]`
    and `vtcache [n_layer, rows_cap, n_kv, 128, tcap]` for rows `[0, rows)`."""
    lib = _lib.load()
    n_layer, _, n_kv, tcap = kcache.shape[:4]
    _lib.check(lib, lib.sv_op_beam_kv_copy(_p(kcache), _p(vtcache), kcache[0].numel(), n_layer, rows, n_kv, tcap, C.byref(plan),
                                           _stream_ptr(kcache.device)))


def op_kv_gather(ksrc: torch.Tensor, vsrc: torch.Tensor, kdst: torch.Tensor, vdst: torch.Tensor, idx: Optional[torch.Tensor],
                 rows: int, length: int) -> None:
    """One layer's cache-row gather (see sv_op_kv_gather): row r of `kdst [>= rows, n_kv, tcap, 128]` / `vdst [>= rows, n_kv,
    128, tcap]` takes the first `length` positions of source row `idx[r]` (int32 on the device, or None: r)."""
    lib = _lib.load()
    n_kv, tcap = ksrc.shape[1], ksrc.shape[2]
    _lib.check(lib, lib.sv_op_kv_gather(_p(ksrc), _p(vsrc), _p(kdst), _p(vdst), _p(idx), rows, n_kv, tcap, length,
                                        _stream_ptr(ksrc.device)))


def op_session_admit(slots, lens, max_new, seeds, seen: torch.Tensor, out_ids: torch.Tensor, pad_id: int, state: dict) -> dict:
    """One session-admission launch (see sv_op_session_admit) over `seen` uint8 `[S, vocab]` and `out_ids` int32
    `[S, out_stride]` (updated in place); `state` holds the RowState and is updated too: `row_len, row_step, row_active,
    row_max_new, row_seed` (`[S]` each) and `event`."""
    lib = _lib.load()
    S, vocab = seen.shape
    i32p, u64 = C.POINTER(C.c_int32), lambda v: (C.c_uint64 * max(1, len(v)))(*[int(s) & (2 ** 64 - 1) for s in v])
    keys = ("row_len", "row_step", "row_active", "row_max_new")
    arrs = {k: _i32s(state[k]) for k in keys}
    row_seed, event, seed = u64(state["row_seed"]), _i32s([state["event"]]), u64(seeds)
    sl, ln, mn = _i32s(slots), _i32s(lens), _i32s(max_new)
    a = _lib.OpAdmit(k=len(slots), S=S, slot_host=C.cast(sl, i32p), len_host=C.cast(ln, i32p), max_new_host=C.cast(mn, i32p),
                     seed_host=C.cast(seed, C.POINTER(C.c_uint64)), seen=seen.data_ptr(), vocab=vocab, out_ids=out_ids.data_ptr(),
                     out_stride=out_ids.shape[1], pad_id=pad_id, row_seed_host=C.cast(row_seed, C.POINTER(C.c_uint64)),
                     event_host=C.cast(event, i32p))
    for k in keys:
        setattr(a, k + "_host", C.cast(arrs[k], i32p))
    _lib.check(lib, lib.sv_op_session_admit(C.byref(a), _stream_ptr(seen.device)))
    for k in keys:
        state[k] = list(arrs[k])[:S]
    state["row_seed"], state["event"] = list(row_seed)[:S], int(event[0])
    return state


def op_decode_chain(mode: int, layers: Sequence[Dict[str, torch.Tensor]], kcache: torch.Tensor, vtcache: torch.Tensor, pos,
                    n_head: int, n_kv: int, n_positions: int, *, ids: Optional[torch.Tensor] = None,
                    x: Optional[torch.Tensor] = None, wte: Optional[torch.Tensor] = None, wpe: Optional[torch.Tensor] = None,
                    lnf: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, lm_head: Optional[torch.Tensor] = None,
                    rope: Optional[Tuple[torch.Tensor, torch.Tensor]] = None, window: int = 0, ln_eps: float = 1e-5,
                    per_row: bool = False, keep: bool = False, pdl: bool = True, graph: bool = False, tiled: bool = False,
                    parts: int = 0) -> Dict[str, object]:
    """One decode step through `sv_op_decode_chain` (the engine's chain, SV_CHAIN_FUSED or SV_CHAIN_PER_OP) over the
    layers given (dicts of the `_lib.CHAIN_LAYER_FIELDS` tensors), caches `kcache [n_layer, >= B, n_kv, tcap, 128]` /
    `vtcache [n_layer, >= B, n_kv, 128, tcap]` (updated) and positions `pos [B]`.  The input is the embedding of `ids`
    (int32 `[B]`) or `x [B, hidden]`; with `lm_head` (and `lnf`) the tail runs too.  `keep`: every layer's intermediates in
    slots of their own (see sv_op_chain) instead of one buffer per activation.  Returns the activation buffers as
    `[slots, B, width]` tensors (`x`, `ln`, `qkv`, `attn`, `h`), `logits [B, vocab]`, FUSED `amax` (val, idx), and the
    `parts_used` / `pdl_used` the call reports."""
    lib = _lib.load()
    n, B = len(layers), len(pos)
    dev = kcache.device
    L0 = layers[0]
    H, I = L0["proj_w"].shape[0], L0["fc_w"].shape[0]
    qkv_cols = L0["attn_w"].shape[0]
    bf = dict(dtype=torch.bfloat16, device=dev)

    def buf(slots, width):    # NaN-filled: a slot read before it is written shows up
        return torch.full((slots if keep else 1, B, width), float("nan"), **bf)

    out = {"x": buf(2 * n + 1, H), "ln": buf(2 * n + 1, H), "qkv": buf(n, qkv_cols), "attn": buf(n, H), "h": buf(n, I)}
    if x is not None:
        out["x"][0].copy_(x.view(B, H))
    larr = (_lib.OpChainLayer * n)(*[_lib.OpChainLayer(*[L[f].data_ptr() for f in _lib.CHAIN_LAYER_FIELDS]) for L in layers])
    posv = _i32s(pos)
    a = _lib.OpChain(mode=mode, n_layer=n, B=B, per_row=int(per_row), hidden=H, n_inner=I, n_head=n_head, n_kv=n_kv,
                     vocab=(wte if wte is not None else lm_head).shape[0] if (wte is not None or lm_head is not None) else 1, n_positions=n_positions, tcap=kcache.shape[3],
                     window=window, ln_eps=ln_eps, rope=int(rope is not None), layers=larr, layer_stride=kcache.stride(0),
                     pos_host=C.cast(posv, C.POINTER(C.c_int32)), pdl=int(pdl), graph=int(graph), tiled=int(tiled),
                     parts=parts, lm_head_tail=int(lm_head is not None))
    a.kcache, a.vtcache = kcache.data_ptr(), vtcache.data_ptr()
    for name in ("x", "ln", "qkv", "attn", "h"):
        t = out[name]
        setattr(a, name, t.data_ptr())
        setattr(a, name + "_stride", t[0].numel() if keep else 0)
    if ids is not None:
        a.ids = ids.data_ptr()
    for name, t in (("wte", wte), ("wpe", wpe), ("lm_head", lm_head)):
        if t is not None:
            setattr(a, name, t.data_ptr())
    if lnf is not None:
        a.lnf_w, a.lnf_b = lnf[0].data_ptr(), lnf[1].data_ptr()
    if rope is not None:
        a.rope_cos, a.rope_sin = rope[0].data_ptr(), rope[1].data_ptr()
    if lm_head is not None:
        out["logits"] = torch.full((B, lm_head.shape[0]), float("nan"), **bf)
        a.logits = out["logits"].data_ptr()
        if mode == _lib.SV_CHAIN_FUSED:
            nt, rs = lib.sv_op_ring_ntiles(lm_head.shape[0]), lib.sv_op_ring_row_stride(B)
            out["amax"] = (torch.full((nt, rs), float("nan"), dtype=torch.float32, device=dev),
                           torch.full((nt, rs), -1, dtype=torch.int32, device=dev))
            a.amax_val, a.amax_idx = out["amax"][0].data_ptr(), out["amax"][1].data_ptr()
    _lib.check(lib, lib.sv_op_decode_chain(C.byref(a), _stream_ptr(dev)))
    out["parts_used"], out["pdl_used"] = int(a.parts_used), bool(a.pdl_used)
    return out


def flow_buffers(B: int, hidden: int, n_inner: int, n_kv: int, vocab: int, device) -> Dict[str, torch.Tensor]:
    """The seven exchange buffers of the dataflow decode kernel (`sv_op_flow_buffer_bytes`), zeroed: `xa xb qkv att hb` as
    int32 flagged words, `part amax` as int64."""
    lib = _lib.load()
    out = {}
    for i, name in enumerate(_lib.FLOW_BUFFERS):
        n = int(lib.sv_op_flow_buffer_bytes(i, B, hidden, n_inner, n_kv, vocab))
        if n < 0:
            raise ValueError(f"no {name} buffer for B={B} hidden={hidden} n_inner={n_inner} n_kv={n_kv} vocab={vocab}")
        out[name] = torch.zeros(n // (8 if name in ("part", "amax") else 4),
                                dtype=torch.int64 if name in ("part", "amax") else torch.int32, device=device)
    return out


def op_decode_flow(layers: Sequence[Dict[str, torch.Tensor]], kcache: torch.Tensor, vtcache: torch.Tensor, n_head: int,
                   n_kv: int, n_positions: int, *, wte: torch.Tensor, lnf: Tuple[torch.Tensor, torch.Tensor],
                   lm_head: torch.Tensor, x_plain: torch.Tensor, bufs: Dict[str, torch.Tensor], cur_len0: int,
                   wpe: Optional[torch.Tensor] = None, nsteps: int = 1, step0: int = 0, first_plain: bool = True,
                   do_select: bool = False, l2_ahead: int = 0, realloc: bool = True, clear: bool = False,
                   params: Optional[GenerationParams] = None, state: Optional[Dict[str, object]] = None,
                   seen: Optional[torch.Tensor] = None, out_ids: Optional[torch.Tensor] = None,
                   next_ids: Optional[torch.Tensor] = None, logits: Optional[torch.Tensor] = None,
                   ln_eps: float = 1e-5) -> Dict[str, object]:
    """One launch of the dataflow decode kernel through `sv_op_decode_flow` over the layers given (dicts of the
    `_lib.CHAIN_LAYER_FIELDS` tensors), caches `kcache [n_layer, >= B, n_kv, tcap, 128]` / `vtcache [n_layer, >= B, n_kv,
    128, tcap]` (updated), the exchange buffers `bufs` (`flow_buffers`; left holding the last step's flagged words) and
    `x_plain [B, hidden]` (the first step's input with `first_plain`; rewritten by every selection).  With `do_select`,
    `state` (dict step / cur_len / done / unfinished, updated in place), `seen [B, vocab]` uint8, `out_ids [B, stride]` and
    `next_ids [B]` (int32) are the generation state.  Returns `logits [B, vocab]` (the last step's), `state`, and the
    `ncta` / `realloc` the launch ran with."""
    lib = _lib.load()
    n, B, H = len(layers), x_plain.shape[0], x_plain.shape[1]
    dev = kcache.device
    V = lm_head.shape[0]
    p = (params or GenerationParams(max_new_tokens=1 << 30, eos_token_id=None)).to_c()
    if logits is None:
        logits = torch.full((B, V), float("nan"), dtype=torch.bfloat16, device=dev)
    larr = (_lib.OpChainLayer * n)(*[_lib.OpChainLayer(*[L[f].data_ptr() for f in _lib.CHAIN_LAYER_FIELDS]) for L in layers])
    a = _lib.OpFlow(n_layer=n, B=B, hidden=H, n_inner=layers[0]["fc_w"].shape[0], n_head=n_head, n_kv=n_kv, vocab=V,
                    n_positions=n_positions, tcap=kcache.shape[3], ln_eps=ln_eps, layers=larr, layer_stride=kcache.stride(0),
                    nsteps=nsteps, step0=step0, cur_len0=cur_len0, first_plain=int(first_plain), do_select=int(do_select),
                    l2_ahead=l2_ahead, realloc=int(realloc), clear=int(clear), params=p)
    a.wte, a.lnf_w, a.lnf_b, a.lm_head = wte.data_ptr(), lnf[0].data_ptr(), lnf[1].data_ptr(), lm_head.data_ptr()
    if wpe is not None:
        a.wpe = wpe.data_ptr()
    a.kcache, a.vtcache, a.x_plain, a.logits = kcache.data_ptr(), vtcache.data_ptr(), x_plain.data_ptr(), logits.data_ptr()
    for name in _lib.FLOW_BUFFERS:
        setattr(a, name, bufs[name].data_ptr())
    counters = unfinished = None
    if do_select:
        counters = _i32s([state["step"], state["cur_len"], state["done"]])
        unfinished = _i32s(state["unfinished"])
        a.counters_host, a.unfinished_host = C.cast(counters, C.POINTER(C.c_int32)), C.cast(unfinished, C.POINTER(C.c_int32))
        a.seen, a.out_ids, a.next_ids, a.out_stride = seen.data_ptr(), out_ids.data_ptr(), next_ids.data_ptr(), out_ids.shape[1]
    _lib.check(lib, lib.sv_op_decode_flow(C.byref(a), _stream_ptr(dev)))
    if do_select:
        state.update(step=counters[0], cur_len=counters[1], done=counters[2], unfinished=[unfinished[b] for b in range(B)])
    return {"logits": logits, "state": state, "ncta": int(a.ncta_used), "realloc": bool(a.realloc_used)}
