"""Import the UNMODIFIED reference package for the benchmark's reference arm and the eager-GPU comparator.

`oracle/_ref/` is the pip install of the reference checkout made by `__graft_entry__.build()` through oracle/reference_install.py
(git-ignored, it travels with the working tree).  Four third-party packages the reference imports are not installed: their inference
branches are restated in tests/golden/_shims (vector_quantize_pytorch.LFQ / VectorQuantize, memory_efficient_attention_pytorch's
FlashAttentionFunction) or stubbed (accelerate, ema_pytorch: trainer-only imports).  Everything else that runs is the
reference's own code, byte-identical to its checkout (checked by tests/test_abi.py when both are present).
None of this repo's kernels, classes or engine is on this path.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
SHIMS = os.path.join(ROOT, "tests", "golden", "_shims")


def available():
    return os.path.isdir(os.path.join(REF_DIR, "muse_maskgit_pytorch"))


def load(d_text=512):
    """Returns the reference's top-level module with t5 config `synth-<d_text>` pre-seeded (no checkpoint download)."""
    if not available():
        raise RuntimeError("oracle/_ref is missing: run `python -c 'import __graft_entry__ as g; g.build()'` where the reference checkout is")
    import transformers  # noqa: F401  (must be imported BEFORE the accelerate stand-in becomes visible)
    from transformers import T5Config
    for p in (SHIMS, REF_DIR):
        if p not in sys.path:
            sys.path.insert(0, p)
    import muse_maskgit_pytorch as ref
    assert os.path.abspath(ref.__file__).startswith(REF_DIR), ref.__file__
    from muse_maskgit_pytorch import t5 as ref_t5
    ref_t5.T5_CONFIGS[f"synth-{d_text}"] = dict(config=T5Config(d_model=d_text))
    return ref
