"""The im2svg loss (`StarVectorStarCoder.forward(batch)`) without a GPU: text suffixes, truncation, targets and the
aggregation over max_batch groups are fed exact fp32 oracle log-probs through a stub scorer and must reproduce the HF
model's own `labels=` loss.  Also home of the oracle restatement of the reference's loss, used by the GPU tests."""
from types import SimpleNamespace

import pytest
import torch

from oracle.pipeline import OracleStarVector
from starvector_b200.config import dims_tiny
from starvector_b200.modeling import StarVectorStarCoder, _SvgTransformer
from starvector_b200.tokenizer import SyntheticTokenizer
from starvector_b200.weights import synthetic_images, synthetic_state_dict


def oracle_im2svg_loss(o, image, svg_list, tok, max_length, v2=False, return_parts=False):
    """`StarVectorBase.forward(batch)` for im2svg, restated over an oracle model: `embed_im_to_svg`
    (starvector_base.py:150-172; `_get_svg_text` starvector_v1.py:20-22 / starvector_v2.py:49-51; `_tokenize` :108-118;
    `_create_targets` :120-123) then the causal LM with `labels=targets` (:174-194)."""
    conditioning_embeds = o.image_projection(o.image_encoder(image.to(o.dtype)))                       # :153-155
    conditioning_embeds_att = torch.ones(conditioning_embeds.size()[:-1], dtype=torch.long)            # :156
    svg_text = [t + ("<svg-end>" if v2 else "") + tok.eos_token for t in svg_list]                     # :159
    svg_tokens = tok(svg_text, truncation=True, add_special_tokens=True, padding="longest", max_length=max_length,
                     return_tensors="pt")                                                              # :161
    svg_tokens_embeds = o._embed(svg_tokens["input_ids"])                                              # :162
    inputs_embeds = torch.cat([conditioning_embeds, svg_tokens_embeds], dim=1)                         # :164
    ids = svg_tokens["input_ids"]
    svg_targets = ids.masked_fill(ids == tok.pad_token_id, -100)                                       # :166
    empty_targets = torch.ones(conditioning_embeds_att.size(), dtype=torch.long).fill_(-100)           # :167
    targets = torch.cat([empty_targets, svg_targets], dim=1)                                           # :168
    attention_mask = torch.cat([conditioning_embeds_att, svg_tokens["attention_mask"]], dim=1)         # :170
    with torch.no_grad():
        out = o.llm(inputs_embeds=inputs_embeds, attention_mask=attention_mask, labels=targets, use_cache=False)  # :183-190
    if return_parts:
        return out.loss, out.logits, targets
    return out.loss


def explicit_causal_lm_loss(logits, targets):
    """HF's causal-LM loss written out: shift by one, fp32 log-softmax, mean over the non-ignored tokens."""
    lp = torch.log_softmax(logits[:, :-1].float(), dim=-1)
    tg = targets[:, 1:]
    keep = tg != -100
    nll = -lp.gather(-1, tg.clamp(min=0).unsqueeze(-1)).squeeze(-1)
    return (nll * keep).sum() / keep.sum()


@pytest.fixture(scope="module")
def tiny():
    d = dims_tiny(max_batch=2)
    sd = synthetic_state_dict(d, seed=3, init="randomized")
    o = OracleStarVector(d, sd, dtype=torch.float32, pad_token_id=d.vocab - 4)
    return d, o


def _facade(o, d, max_length, max_batch, v2=False):
    """The loss path of StarVectorStarCoder with the engine replaced by a stub scorer over the fp32 oracle."""
    m = StarVectorStarCoder.__new__(StarVectorStarCoder)
    m.v2, m.max_length, m.llm_config = v2, max_length, {}
    m.svg_transformer = _SvgTransformer(m, SyntheticTokenizer(d.vocab, n_added=5 if v2 else 4))
    m.engine = SimpleNamespace(dims=SimpleNamespace(max_batch=max_batch))
    calls = []

    def score_group(image, svg_ids):
        calls.append(svg_ids.shape[0])
        with torch.no_grad():
            prefix = o.image_projection(o.image_encoder(image.to(o.dtype)))
            emb = torch.cat([prefix, o._embed(svg_ids)], dim=1)
            logits = o.llm(inputs_embeds=emb, use_cache=False).logits[:, prefix.shape[1] - 1:-1].float()
        return torch.log_softmax(logits, dim=-1).gather(-1, svg_ids.unsqueeze(-1)).squeeze(-1)

    m._score_group = score_group
    return m, calls


SVGS = ["<t11><t12><t13><t14><t15><t16><t17>", "<t21><t22>", "<t31><t32><t33><t34><t35>"]


def test_oracle_restatement_equals_explicit_loss(tiny):
    d, o = tiny
    tok = SyntheticTokenizer(d.vocab)
    img = synthetic_images(d, 3, seed=5)
    loss, logits, targets = oracle_im2svg_loss(o, img, SVGS, tok, max_length=6, return_parts=True)
    assert targets.shape[1] == d.query_length + 6                                # truncated to max_length
    assert abs(float(loss) - float(explicit_causal_lm_loss(logits, targets))) < 1e-6


@pytest.mark.parametrize("max_batch", [8, 2])
def test_loss_assembly_matches_hf_labels_loss(tiny, max_batch):
    d, o = tiny
    img = synthetic_images(d, 3, seed=5)
    for max_length in (6, 64):                                                  # truncating and not
        m, calls = _facade(o, d, max_length, max_batch)
        got = float(m.forward({"image": img, "svg": SVGS}))
        ref = float(oracle_im2svg_loss(o, img, SVGS, m.svg_transformer.tokenizer, max_length))
        assert abs(got - ref) < 1e-6, (max_length, got, ref)
        assert calls == ([3] if max_batch >= 3 else [2, 1])


def test_svg_text_suffixes():
    d = dims_tiny()
    for v2, want in ((False, ["a<|endoftext|>"]), (True, ["a<svg-end><|endoftext|>"])):
        m = StarVectorStarCoder.__new__(StarVectorStarCoder)
        m.v2, m.llm_config = v2, {}
        m.svg_transformer = _SvgTransformer(m, SyntheticTokenizer(d.vocab, n_added=5 if v2 else 4))
        assert m._get_svg_text(["a"]) == want
    tok = SyntheticTokenizer(d.vocab, n_added=5)
    assert tok("<t3><svg-end><|endoftext|>")["input_ids"] == [3, tok.pad_token_id + 4, tok.eos_token_id]


def test_v2_unequal_lengths_raise(tiny):
    d, o = tiny
    m, calls = _facade(o, d, 64, 8, v2=True)
    with pytest.raises(NotImplementedError):
        m.forward({"image": synthetic_images(d, 2, seed=5), "svg": SVGS[:2]})
    assert calls == []
