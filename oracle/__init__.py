"""CPU oracle for the im2svg hot path — TEST INFRASTRUCTURE ONLY.

Nothing under ``oracle/`` is part of the product: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import it, and only as the checker / the timed CPU baseline.  The product path
(`starvector_b200`) never imports this package and fails loudly if its CUDA library is
missing.

What the oracle is: a CPU restatement of the reference's ``generate_im2svg`` path
(reference: starvector/model/models/starvector_base.py:203-259) around
  * a functional restatement of the in-tree CLIP ViT (clip_model.py:117-191,
    image_encoder.py:50-61,91-94) and Adapter (adapters/adapter.py:5-39), and
  * the *installed* ``transformers`` ``GPTBigCodeForCausalLM`` + ``GenerationMixin.generate``
    (the reference loads that class by name: llm/starcoder.py:33; pinned 4.49.0,
    installed 5.5.0 — drift recorded in DESIGN.md).

Parity pinning: the reference has NO tests/golden vectors for this path (SURVEY.md §4,
§8c).  The restatement is pinned instead against outputs of the reference's own modules
(`oracle/make_golden.py` imports ``starvector/...`` from a checkout of the reference and
writes ``tests/golden/*.pt``); see
``tests/test_oracle_golden.py``.
"""
