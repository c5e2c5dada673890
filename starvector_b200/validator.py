"""Engine-backed backend for the reference's validation harness (SURVEY.md §3.2, §8f-4).

Reference contract this module honours:
  * validators are `SVGValidator` subclasses registered with `@register_validator`
    (starvector/validation/svg_validator_base.py:19-26) and picked by `config.model.generation_engine`
    (starvector/validation/validate.py:8-12, full class names are accepted as they are);
  * the HF backend builds the model, takes `tokenizer` / `svg_end_token_id` from it
    (starvector_hf_validator.py:43-60), provides `get_dataloader`, `release_memory` and
    `generate_svg(batch, generate_config)` (:77-88): temperature 0 means greedy, images go to the device in the
    configured dtype, then `self.model.model.generate_im2svg(batch=batch, **generate_config)` returns the strings the
    base class post-processes (svg_validator_base.py:373-377).

`register()` imports the reference's registry (the reference must be importable: `pip install -e` of joanrod/star-vector
or its checkout on `sys.path`) and registers `StarVectorB200Validator`, so `generation_engine: StarVectorB200Validator`
(or the short name `b200` after `install_short_name`) selects this engine.  Without the reference, `B200GenerateMixin`
is still usable on its own (tests/test_validator.py drives it with a stand-in base class).
"""
from __future__ import annotations

from typing import Any, Dict, List, Mapping

import torch

ENGINE_NAME = "StarVectorB200Validator"


class B200GenerateMixin:
    """The model-facing half of `StarVectorHFSVGValidator` (starvector_hf_validator.py:43-88) on the H100 engine."""

    def init_engine(self, config) -> None:
        """`config`: the harness' omegaconf tree (model.name / model.from_checkpoint / model.torch_dtype / run.device)."""
        from .modeling import StarVectorForCausalLM

        self.torch_dtype = {"bfloat16": torch.bfloat16, "float16": torch.float16, "float32": torch.float32}[config.model.torch_dtype]
        path = getattr(self, "resume_from_checkpoint", None) if config.model.from_checkpoint else config.model.name   # :55-58
        batch_size = int(getattr(config.dataset, "batch_size", 8))
        num_beams = max(1, int(getattr(config.generation_params, "num_beams", 2)))   # generate_im2svg's default (:234)
        max_len = int(getattr(config.generation_params, "max_length", 8192))
        # beams are cache rows: size the engine for a whole batch of beams when it fits the 16 rows a GPU holds
        self.model = StarVectorForCausalLM.from_pretrained(path, torch_dtype=self.torch_dtype, max_batch=min(batch_size * num_beams, 16),
                                                           max_len=max_len)
        self.bind_model(self.model)

    def bind_model(self, model) -> None:
        self.model = model
        self.processor = model.model.processor                                    # SVGValDataset applies it per sample (:30-33)
        self.tokenizer = model.model.svg_transformer.tokenizer                    # :59
        self.svg_end_token_id = self.tokenizer("</svg>", add_special_tokens=False)["input_ids"][0]   # :60

    def generate_svg(self, batch: Dict[str, Any], generate_config: Mapping[str, Any]) -> List[str]:
        """starvector_hf_validator.py:77-88, statement for statement."""
        generate_config = dict(generate_config)                                   # the reference mutates its DictConfig in place
        if generate_config.get("temperature") == 0:
            generate_config["temperature"] = 1.0
            generate_config["do_sample"] = False
        batch["image"] = batch["image"].to(self.model.device).to(torch.bfloat16)  # the engine computes in bf16 (DESIGN.md §7)
        if self.task == "im2svg":
            return self.model.model.generate_im2svg(batch=batch, **generate_config)
        raise NotImplementedError(f"task {self.task!r}: generate_text2svg raises TypeError in the reference itself "
                                  "(starvector_base.py:320-323 calls a one-argument method with two)")

    def release_memory(self) -> None:                                             # :66-75
        if getattr(self, "model", None) is not None:
            self.model.model.engine.close()
            self.model = None
        if torch.cuda.is_available():
            torch.cuda.empty_cache()


def make_validator_class(base_cls, register_validator=None):
    """`StarVectorB200Validator(base_cls)`; `register_validator` = the reference's decorator (or None)."""

    class StarVectorB200Validator(B200GenerateMixin, base_cls):
        def __init__(self, config):
            base_cls.__init__(self, config)
            self.init_engine(config)
            if hasattr(self, "get_dataloader"):
                self.get_dataloader()

    StarVectorB200Validator.__name__ = StarVectorB200Validator.__qualname__ = ENGINE_NAME
    return register_validator(StarVectorB200Validator) if register_validator else StarVectorB200Validator


def register():
    """Register with the reference's own registry; returns the class.  Raises ImportError when the reference is absent."""
    from starvector.validation import svg_validator_base as ref                  # noqa: the reference package

    if ENGINE_NAME in ref.validator_registry:
        return ref.validator_registry[ENGINE_NAME]
    return make_validator_class(ref.SVGValidator, ref.register_validator)


def install_short_name(validate_module, short: str = "b200") -> None:
    """`generation_engine: b200` — validate.py builds its ENGINE_MAPPING inside `get_validator`, so the short name is added
    by wrapping that function (the full class name needs nothing)."""
    inner = validate_module.get_validator

    def get_validator(validator_name, config):
        if str(config.model.generation_engine).lower() == short:
            config.model.generation_engine = ENGINE_NAME
        return inner(validator_name, config)

    validate_module.get_validator = get_validator
