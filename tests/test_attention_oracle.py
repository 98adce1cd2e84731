"""The attention oracle checked against itself on the CPU: the reference against torch's scaled_dot_product_attention, the clean emulation of
the wgmma kernel's rounding inside the bf16 tolerance, and every injected defect outside it on the probe cases."""
import pytest
import torch
import torch.nn.functional as F

from tests import attention_oracle as A

torch.set_grad_enabled(False)

# (B, heads, Tq, Tk, mask kind, scale, logit_bound): both block sizes, full and ragged tails, both softmax modes, every mask family
FAMILIES = [
    (3, 3, 40, 2, None, 8.0, 0.0),
    (3, 3, 40, 34, "sweep", 8.0, 1.02),
    (3, 3, 130, 65, None, 8.0, 1.02),
    (3, 3, 130, 98, "sweep", 8.0, 0.0),
    (2, 3, 130, 290, "random", 8.0, 0.0),
    (2, 3, 70, 290, "only_last", 8.0, 1.02),
    (2, 3, 70, 290, "only_first", 1.0, 0.0),
    (3, 2, 70, 257, "chunk_dead", 8.0, 1.02),
    (3, 2, 70, 257, "per_entry", 32.0, 0.0),
    (3, 2, 70, 257, "first_entry_dead", 8.0, 20.0),
    (3, 3, 130, 641, "sweep", 8.0, 1.02),
    (3, 3, 130, 642, None, 8.0, 0.0),
    (3, 3, 40, 737, "sweep", 8.0, 0.0),
    (2, 3, 40, 1025, None, 8.0, 1.02),
]


def _fid(c):
    return f"B{c[0]}h{c[1]}-q{c[2]}-k{c[3]}-{c[4] or 'nomask'}-s{c[5]:g}-b{c[6]:g}"


def _case(c, probe=True):
    B, H, Tq, Tk, kind, scale, bound = c
    q, k, v = A.operands(_fid(c), B, H, Tq, Tk, True, probe=probe)
    return q, k, v, A.mask_of(kind, _fid(c), B, Tk), scale, bound


@pytest.mark.parametrize("c", FAMILIES, ids=[_fid(c) for c in FAMILIES])
def test_clean_emulation_is_inside_the_bf16_tolerance(c):
    q, k, v, mask, scale, bound = _case(c)
    ref, w = A.reference(q, k, v, mask, scale)
    got = A.emulate_bf16(q, k, v, mask, scale, logit_bound=bound)
    variant = A.TC64 if A.block_plan(c[3] - 1)[0] == 64 else A.TC128
    r = A.worst_ratio(got, ref, A.tolerance(variant, ref, w, scale))
    print(f"{variant}: worst err / tol {r:.3f}")
    assert r <= 1.0, r
    if mask is not None and not bool(mask[0].any()):                      # a fully masked entry is the null value, bit for bit
        assert torch.equal(got[0], v[0, :, :1].expand(-1, c[2], -1))


# the probe cases a defect has to be caught on: a masked and an unmasked one per block size, with a ragged tail
PROBES = [c for c in FAMILIES if c[3] in (98, 290, 641, 737) and c[4] in ("sweep", "random")] + [(3, 3, 130, 98, None, 8.0, 0.0), (3, 3, 130, 737, None, 8.0, 1.02)]
NEEDS_MASK = ("mask_shift_by_one", "mask_row_of_wrong_batch")


@pytest.mark.parametrize("defect", A.DEFECTS)
def test_every_injected_defect_is_rejected(defect):
    caught = 0
    for c in PROBES:
        if defect in NEEDS_MASK and c[4] is None:
            continue
        q, k, v, mask, scale, bound = _case(c)
        ref, w = A.reference(q, k, v, mask, scale)
        variant = A.TC64 if A.block_plan(c[3] - 1)[0] == 64 else A.TC128
        r = A.worst_ratio(A.emulate_bf16(q, k, v, mask, scale, logit_bound=bound, defect=defect), ref, A.tolerance(variant, ref, w, scale))
        print(f"{defect} on {_fid(c)}: worst err / tol {r:.1f}")
        assert r > 2.0, f"{defect} passes on {_fid(c)} (worst err / tol {r:.3f})"
        caught += 1
    assert caught >= 2


def test_what_the_old_rule_accepted():
    """a report (printed); the one acceptance the oracle's module docstring states is pinned"""
    table = A.old_rule_accepts()
    for name, row in table.items():
        print(name + ": " + ", ".join(f"{d} {'ACCEPTED' if ok else 'rejected'}" for d, ok in row.items()))
    assert table["unmasked 256x257"]["normalise_without_null"] and table["unmasked 1024x1025"]["normalise_without_null"]


def test_reference_agrees_with_sdpa():
    B, H, Tq, Tk, scale = 3, 2, 9, 41, 5.0
    q, k, v = A.operands("sdpa", B, H, Tq, Tk, False)
    mask = A.mask_of("first_entry_dead", "sdpa", B, Tk)
    ref, w = A.reference(q, k, v, mask, scale)
    live = F.pad(mask, (1, 0), value=True)[:, None, None, :].expand(B, H, Tq, Tk)
    want = F.scaled_dot_product_attention(q.double(), k.double(), v.double(), attn_mask=live, scale=scale)
    assert float((ref - want).abs().max()) < 1e-12
    assert bool((w >= ref.abs() - 1e-12).all())
    # one K / V per head, broadcast over the batch
    q, k, v = A.operands("sdpa.shared", B, H, Tq, Tk, False, kv_shared=True)
    ref, _ = A.reference(q, k, v, mask, scale)
    want = F.scaled_dot_product_attention(q.double(), k.double().expand(B, -1, -1, -1), v.double().expand(B, -1, -1, -1), attn_mask=live, scale=scale)
    assert float((ref - want).abs().max()) < 1e-12


def test_block_plan_and_probes():
    assert A.block_plan(1) == (64, 1, 32) and A.block_plan(64) == (64, 1, 64) and A.block_plan(65) == (64, 2, 32)
    assert A.block_plan(640) == (64, 10, 64) and A.block_plan(641) == (128, 6, 32) and A.block_plan(736) == (128, 6, 96)
    assert A.block_plan(1024) == (128, 8, 128) and A.block_plan(4095) == (128, 32, 128)
    assert A.single_pass(8.0, 1.02) and A.single_pass(8.0, 4.3) and not A.single_pass(8.0, 20.0) and not A.single_pass(8.0, 0.0)
    assert A.probe_keys(737)[:5] == [0, 1, 736, 641, 640]
