"""CPU: libmmg.so builds for sm_90a, loads without a GPU/driver, exports every symbol include/mmg.h declares, and the
ctypes mirror of every argument block has the C struct's size.  No compute calls here."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_header_symbols():
    from muse_maskgit_pytorch_b200 import build, _lib
    build.build()
    header = open(os.path.join(ROOT, "include", "mmg.h")).read()
    declared = set(re.findall(r"^\s*(?:int|int64_t|uint64_t|const char\*)\s+(mmg_[a-z0-9_]+)\s*\(", header, re.M))
    assert {"mmg_linear", "mmg_attention", "mmg_logits_sample", "mmg_vq_lfq_encode", "mmg_vq_l2_argmin", "mmg_conv2d",
            "mmg_conv_transpose2d", "mmg_remask", "mmg_version"} <= declared
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in mmg.h but not exported"
    assert set(_lib.EXPORTS) | set(_lib.PLAIN_EXPORTS) == declared
    assert _lib.lib().mmg_version() == 101          # also runs the struct-size self check


def test_ops_fail_loudly_without_library(monkeypatch, tmp_path):
    from muse_maskgit_pytorch_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "missing.so"))
    try:
        _lib.lib()
    except _lib.MMGError as e:
        assert "no fallback" in str(e)
    else:
        raise AssertionError("missing library must raise")


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "muse_maskgit_pytorch_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "oracle" not in src.replace("# oracle", ""), f"{fn} references the oracle"


def test_state_dict_keys_match_reference_tables():
    """Checkpoint-key contract (SURVEY.md 8b): our parameter holders expose exactly the reference's keys/shapes
    (oracle/shapes.py is asserted against the unmodified reference in tests/golden/make_golden.py)."""
    import muse_maskgit_pytorch_b200 as M
    from muse_maskgit_pytorch_b200 import t5
    from oracle import shapes
    t5.T5_CONFIGS["synth-96"] = {"d_model": 96}
    tr = M.MaskGitTransformer(num_tokens=1024, dim=128, seq_len=16, depth=2, heads=2, t5_name="synth-96")
    got = {k: tuple(v.shape) for k, v in tr.state_dict().items()}
    assert got == {k: tuple(v) for k, v in shapes.transformer_shapes(1024, 128, 16, 2, heads=2, text_dim=96).items()}
    vae = M.VQGanVAE(dim=64, codebook_size=512)
    got = {k: tuple(v.shape) for k, v in vae.state_dict().items() if k != "quantizer.mask"}
    assert got == {k: tuple(v) for k, v in shapes.vae_shapes(64, codebook_size=512).items()}
    assert "quantizer.mask" in vae.state_dict()
    critic = M.TokenCritic(num_tokens=1024, dim=128, seq_len=16, depth=1, heads=2, t5_name="synth-96")
    assert critic.state_dict()["to_logits.weight"].shape == (1, 128) and critic.mask_id is None


def test_decode_step_workspace_query_is_host_only():
    """mmg_decode_step_workspace_bytes is pure host arithmetic: callable without a GPU, grows with the logits buffer."""
    from muse_maskgit_pytorch_b200 import _lib
    f = _lib.lib().mmg_decode_step_workspace_bytes
    c3 = f(64, 2, 256, 512, 8, 1408, 65536, 256)
    assert c3 >= 64 * 256 * 65536 * 4 and c3 % 256 == 0
    assert f(8, 2, 256, 512, 8, 1408, 65536, 256) < c3 and f(0, 2, 256, 512, 8, 1408, 65536, 256) == 0


def test_fused_logits_planner_restatement_matches_workspace_query():
    """oracle/fused_tail.py's restatement of mmg_logits_fused's planner (split count S and list capacity per row count, on the SM count the
    library sees: the device's, or 132 without one) gives the library's workspace size everywhere: the GPU tests choose their row counts
    from it to reach given plans."""
    import math
    import torch
    from muse_maskgit_pytorch_b200 import ops
    from oracle import fused_tail as FT
    units = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    for V in (1024, 1280, 4096, 8192, 12288, 65536):
        for K in (64, 512, 1024):
            for k in (math.ceil(0.1 * V), math.ceil(0.2 * V)):
                for R in (1, 77, 128, 129, 300, 1000, 2048, 4097, 6912, 8192, 8300, 13952, 16384, 16385, 25000, 40000):
                    assert FT.workspace_bytes(R, V, K, k, units) == ops.logits_fused_workspace_bytes(R, V, K, k), (R, V, K, k, units)
    assert FT.workspace_bytes(300, 65536, 512, math.ceil(0.2 * 65536), units) == 0
    assert FT.lf_plan(16384, 65536, 132)["S"] == 1 and FT.lf_plan(8192, 65536, 132)["S"] == 2
    for sms in (132, 114):                 # H100 SXM / PCIe: the GPU tests reach the shared-segment plans S = 1, 2 at V = 65536 on both
        assert FT.rows_for_plan(65536, 1, sms) and FT.rows_for_plan(65536, 2, sms)


def test_baseline_ref_is_the_unmodified_reference():
    """oracle/_ref (the reference arm of bench.py) is byte-identical to the reference checkout wherever both exist."""
    import filecmp
    import pytest
    from oracle import reference_install as RI
    src = RI.source_dir()
    inst = os.path.join(RI.DEST, RI.PACKAGE)
    if src is None or not RI.installed():
        pytest.skip("needs the reference checkout and oracle/_ref")
    ref = os.path.join(src, RI.PACKAGE)
    names = sorted(f for f in os.listdir(ref) if f.endswith(".py"))
    assert names and names == sorted(f for f in os.listdir(inst) if f.endswith(".py"))
    match, mismatch, errors = filecmp.cmpfiles(ref, inst, names, shallow=False)
    assert not mismatch and not errors, (mismatch, errors)


def test_pack_cache_digest_tracks_weights():
    """The on-disk pre-pack cache key (pack_cache.weights_digest) is a function of names, shapes, dtypes and bytes of the module's tensors."""
    import torch
    from muse_maskgit_pytorch_b200 import pack_cache
    torch.manual_seed(0)
    a, b = torch.nn.Linear(8, 4), torch.nn.Linear(8, 4)
    b.load_state_dict(a.state_dict())
    assert pack_cache.weights_digest(a, ("bf16",)) == pack_cache.weights_digest(b, ("bf16",))
    assert pack_cache.weights_digest(a, ("bf16",)) != pack_cache.weights_digest(a, ("fp32",))
    with torch.no_grad():
        b.weight[0, 0] += 1e-3
    assert pack_cache.weights_digest(a, ("bf16",)) != pack_cache.weights_digest(b, ("bf16",))
