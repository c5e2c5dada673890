"""Model/configuration records for the H100 im2svg engine.

`StarVectorConfig` mirrors the field names and defaults of the reference's
``StarVectorConfig`` (reference: starvector/model/starvector_arch.py:96-131) so a
``config.json`` written by the reference loads unchanged.  `ModelDims` is the flat
record of integers the C-ABI (`include/starvector_b200.h`, ``sv_model_desc``) takes.
Dimension sources: SURVEY.md §8 (image_encoder.py:50-61, starvector_base.py:87-104).
"""
from __future__ import annotations

import dataclasses
import json
import os
from typing import Any, Dict


@dataclasses.dataclass
class ModelDims:
    """Everything the engine needs to size kernels and buffers (all ints/floats)."""

    variant: int = 0              # 0 = v1 (CLIP ViT + GPTBigCode MQA); 1 = v2 (SigLIP + StarCoder2)
    # vision tower (clip_model.py:167-179, image_encoder.py:50-61)
    image_size: int = 224
    patch_size: int = 14
    vit_width: int = 1024
    vit_layers: int = 23
    vit_heads: int = 16
    vit_mlp: int = 4096
    # adapter (adapter.py:13-31)
    adapter_norm: int = 0         # 0 = layer_norm over [Q,H]; 1 = BatchNorm1d(Q) eval
    # decoder (bigcode/starcoderbase-1b; SURVEY.md §8)
    hidden: int = 2048
    n_layer: int = 24
    n_head: int = 16
    n_kv_head: int = 1
    head_dim: int = 128
    n_inner: int = 8192
    n_positions: int = 8192
    vocab: int = 49156
    ln_eps: float = 1e-5
    # engine capacity
    max_batch: int = 8            # cache rows (images x beams / completions) per GPU, 1..16
    max_len: int = 8192           # KV-cache capacity in tokens (<= n_positions for v1)
    # v2 (SigLIP + StarCoder2) only
    rope_theta: float = 0.0       # 0 = learned absolute positions (v1)
    sliding_window: int = 0
    vit_ln_eps: float = 1e-5

    @property
    def query_length(self) -> int:
        # CLIP prepends a class token (clip_model.py:185); SigLIP does not (starvector_base.py:99-104: 576 @384)
        return (self.image_size // self.patch_size) ** 2 + (1 if self.variant == 0 else 0)

    @property
    def patch_k(self) -> int:
        return 3 * self.patch_size * self.patch_size

    @property
    def patch_k_padded(self) -> int:
        return (self.patch_k + 63) // 64 * 64

    def decoder_weight_bytes(self) -> int:
        """Bytes of bf16 decoder weights streamed per decode step (SURVEY.md §8d `W`)."""
        h, i, kv = self.hidden, self.n_inner, self.n_kv_head * self.head_dim
        per_layer = (  # identical parameter count for GPTBigCode (packed c_attn) and StarCoder2 (q/k/v/o + biases)
            2 * h + (h + 2 * kv) * h + (h + 2 * kv)      # ln_1, c_attn
            + h * h + h                                   # attn.c_proj
            + 2 * h + i * h + i + h * i + h               # ln_2, mlp
        )
        return 2 * (self.n_layer * per_layer + 2 * h + self.vocab * h)

    def kv_bytes_per_token(self) -> int:
        return self.n_layer * 2 * self.n_kv_head * self.head_dim * 2


def dims_1b(max_batch: int = 8, max_len: int = 8192) -> ModelDims:
    """StarVector-1B: CLIP ViT-L/14@224 (23 blocks) + starcoderbase-1b."""
    return ModelDims(max_batch=max_batch, max_len=max_len)


def dims_8b(max_batch: int = 4, max_len: int = 16384, rope_theta: float = 1.0e6) -> ModelDims:
    """StarVector-8B: SigLIP-L/16@384 (24 blocks, 576 tokens) + starcoder2-7b (36 q / 4 kv heads, RoPE, SWA 4096).

    Dimensions from SURVEY.md §8 (configs/models/starvector-8b/im2svg-stack.yaml, modeling_siglip / modeling_starcoder2);
    `rope_theta` comes from the hub config of bigcode/starcoder2-7b, which is not available offline: pass the real value.
    """
    return ModelDims(
        variant=1, image_size=384, patch_size=16, vit_width=1024, vit_layers=24, vit_heads=16, vit_mlp=4096,
        hidden=4608, n_layer=32, n_head=36, n_kv_head=4, head_dim=128, n_inner=18432, n_positions=16384, vocab=49157,
        ln_eps=1e-5, max_batch=max_batch, max_len=max_len, rope_theta=rope_theta, sliding_window=4096, vit_ln_eps=1e-6,
    )


def refine_dims_from_state_dict(d: ModelDims, sd) -> ModelDims:
    """Decoder dimensions as the CHECKPOINT has them (tensor shapes win over config fields): a v1 checkpoint whose
    `max_length` differs from the decoder's `n_positions`, or any model size other than 1B / 8B, loads instead of
    failing with a shape mismatch.  Only fields that a tensor shape determines are touched."""
    v2 = d.variant == 1
    pre = "model.svg_transformer.transformer." + ("model." if v2 else "transformer.")
    emb = sd.get(pre + ("embed_tokens.weight" if v2 else "wte.weight"))
    if emb is None:
        return d
    over = {"vocab": int(emb.shape[0]), "hidden": int(emb.shape[1])}
    layer = pre + ("layers." if v2 else "h.")
    over["n_layer"] = 1 + max(int(k[len(layer):].split(".")[0]) for k in sd if k.startswith(layer))
    fc = sd.get(layer + "0.mlp.c_fc.weight")
    if fc is not None:
        over["n_inner"] = int(fc.shape[0])
    over["n_head"] = over["hidden"] // d.head_dim
    if v2:
        kp = sd.get(layer + "0.self_attn.k_proj.weight")
        if kp is not None:
            over["n_kv_head"] = int(kp.shape[0]) // d.head_dim
    else:
        wpe = sd.get(pre + "wpe.weight")
        if wpe is not None:
            over["n_positions"] = int(wpe.shape[0])
    out = dataclasses.replace(d, **over)
    out.max_len = min(out.max_len, out.n_positions)
    return out


def dims_tiny_v2(max_batch: int = 4, max_len: int = 192, **over) -> ModelDims:
    """Few-MB model with the 8B family's structure (SigLIP tower, GQA group 2, RoPE, sliding window 24)."""
    d = ModelDims(
        variant=1, image_size=64, patch_size=16, vit_width=128, vit_layers=2, vit_heads=2, vit_mlp=512,
        hidden=512, n_layer=2, n_head=4, n_kv_head=2, head_dim=128, n_inner=1024, n_positions=192, vocab=500,
        ln_eps=1e-5, max_batch=max_batch, max_len=max_len, rope_theta=10000.0, sliding_window=24, vit_ln_eps=1e-6,
    )
    return dataclasses.replace(d, **over)


def dims_tiny(max_batch: int = 4, max_len: int = 256, **over) -> ModelDims:
    """A few-MB model with the same structure, for parity tests the oracle finishes in seconds."""
    d = ModelDims(
        image_size=56, patch_size=14, vit_width=128, vit_layers=2, vit_heads=2, vit_mlp=512,
        hidden=256, n_layer=2, n_head=2, n_kv_head=1, head_dim=128, n_inner=1024,
        n_positions=256, vocab=500, max_batch=max_batch, max_len=max_len,
    )
    return dataclasses.replace(d, **over)


class StarVectorConfig:
    """Field-compatible stand-in for the reference's PretrainedConfig subclass.

    (reference: starvector/model/starvector_arch.py:96-131).  Kept free of a
    `transformers` dependency so importing the engine never touches the hub.
    """

    model_type = "starvector"

    def __init__(
        self,
        starcoder_model_name: str = "bigcode/starcoderbase-1b",
        image_encoder_type: str = "clip",
        adapter_norm: str = "layer_norm",
        image_size: int = 224,
        max_length: int = 8192,
        max_length_train: int = 8192,
        use_flash_attn: bool = True,
        use_cache: bool = True,
        num_attention_heads: int = 16,
        num_hidden_layers: int = 24,
        vocab_size: int = 49152,
        hidden_size: int = 2048,
        num_kv_heads: int = 4,
        torch_dtype: str = "bfloat16",
        **kwargs: Any,
    ) -> None:
        self.starcoder_model_name = starcoder_model_name
        self.image_encoder_type = image_encoder_type
        self.adapter_norm = adapter_norm
        self.image_size = image_size
        self.max_length = max_length
        self.max_length_train = max_length_train
        self.use_flash_attn = use_flash_attn
        self.use_cache = use_cache
        self.num_attention_heads = num_attention_heads
        self.num_hidden_layers = num_hidden_layers
        self.vocab_size = vocab_size
        self.hidden_size = hidden_size
        self.num_kv_heads = num_kv_heads
        self.torch_dtype = torch_dtype
        self._name_or_path = kwargs.pop("_name_or_path", "")
        # engine-side extras (not in the reference): explicit dims for synthetic/tiny models
        self.engine_dims: Dict[str, Any] = dict(kwargs.pop("engine_dims", {}) or {})
        self.extra = kwargs

    # -- (de)serialisation compatible with a reference `config.json` ---------------------
    def to_dict(self) -> Dict[str, Any]:
        d = {k: v for k, v in self.__dict__.items() if k not in ("extra",)}
        d["model_type"] = self.model_type
        return d

    @classmethod
    def from_json_file(cls, path: str) -> "StarVectorConfig":
        with open(path) as f:
            d = json.load(f)
        d.pop("model_type", None)
        d.pop("architectures", None)
        d.pop("auto_map", None)
        return cls(**d)

    @classmethod
    def from_pretrained(cls, path: str) -> "StarVectorConfig":
        cfg = os.path.join(path, "config.json")
        if not os.path.isfile(cfg):
            raise FileNotFoundError(
                f"{cfg} not found: this build has no network access; pass a local checkpoint "
                "directory or construct the model with StarVectorForCausalLM.from_config()."
            )
        c = cls.from_json_file(cfg)
        c._name_or_path = path
        return c

    def to_dims(self, max_batch: int = 8, max_len: int | None = None) -> ModelDims:
        """Resolve kernel dimensions: v1 = CLIP + GPTBigCode, v2 ('starcoder2' in the name, starvector_arch.py:137-145)
        = SigLIP + StarCoder2."""
        if "starcoder2" in self.starcoder_model_name:
            if "siglip" not in self.image_encoder_type:
                raise NotImplementedError(f"image_encoder_type={self.image_encoder_type!r}: v2 is built for siglip towers")
            d = dims_8b(max_batch=max_batch, max_len=max_len or self.max_length)
            d.image_size = self.image_size if self.image_size != 224 else 384
            d.adapter_norm = {"layer_norm": 0, "batch_norm": 1}[self.adapter_norm]
            if self.engine_dims:
                d = dataclasses.replace(d, **self.engine_dims)
            d.max_len = min(d.max_len, d.n_positions)
            return d
        if self.image_encoder_type != "clip":
            raise NotImplementedError(f"image_encoder_type={self.image_encoder_type!r}: only 'clip' is built for v1")
        d = ModelDims(
            image_size=self.image_size,
            hidden=self.hidden_size,
            n_layer=self.num_hidden_layers,
            n_head=self.num_attention_heads,
            head_dim=self.hidden_size // self.num_attention_heads,
            n_inner=4 * self.hidden_size,
            n_positions=self.max_length,
            # tokenizer adds [PAD] + 3 tokens (llm/starcoder.py:43-53) then resize_token_embeddings
            vocab=self.vocab_size + 4 if self.vocab_size == 49152 else self.vocab_size,
            adapter_norm={"layer_norm": 0, "batch_norm": 1}[self.adapter_norm],
            max_batch=max_batch,
            max_len=max_len or self.max_length,
        )
        if self.engine_dims:
            d = dataclasses.replace(d, **self.engine_dims)
        d.max_len = min(d.max_len, d.n_positions)
        return d
