"""GPU parity tests of the fused to_logits + sampling tail (mmg_logits_fused: no [rows, V] logits buffer) against the materialised path
(mmg_linear + mmg_logits_sample, itself pinned to the oracle in test_gpu_kernels.py): same token ids, same scores up to the summation order
of the softmax denominator, for libmmg's Philox keying, injected noise and the ATen stream; rows whose sampled threshold cannot work
(constant logits) take the in-call fallback; too many of them raise the overflow word and generate() repeats on the materialised path.
Beyond parity: every split plan class (S = 1 and 2, whose finisher shares a list segment among warps, up to the largest S) against an fp64
oracle, hand-built rows for each fallback reason and the exclusion loop, one workspace across a mask schedule, only_masked, and the
MMG_FINISH_MINB=6 finisher build."""
import math
import os
import subprocess
import sys

import pytest
import torch

from oracle import fused_tail as FT, philox, muse_oracle as O
from tests import util

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
bf = torch.bfloat16


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def _case(R, V, K, seed, b=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    e = torch.randn((R, K), generator=g, device="cuda").to(bf)
    w = (torch.randn((V, K), generator=g, device="cuda") * K ** -0.5).to(bf)
    b = b or 1
    assert R % b == 0
    nm = R // b
    n = nm + 3
    mp = torch.stack([torch.sort(torch.randperm(n, generator=g, device="cuda")[:nm]).values for _ in range(b)]).int().contiguous()
    return e, w, b, n, nm, mp


def _run_both(e, w, b, n, nm, mp, k, temp, ws=None, status=None, rows_capacity=None, **kw):
    """materialised path (ids_a, sc_a) and fused path (ids_b, sc_b) on the same rows; the fused call gets its own workspace sized for
    exactly these rows unless one (with its rows_capacity) is passed in."""
    o = ops()
    R, V = e.shape[0], w.shape[0]
    ids_a = torch.full((b, n), V, dtype=torch.long, device="cuda"); sc_a = torch.full((b, n), -1e5, device="cuda")
    ids_b, sc_b = ids_a.clone(), sc_a.clone()
    lg = torch.empty((R, V), device="cuda")
    o.linear(e, w, lg)
    o.logits_sample(lg, mp, ids_a, sc_a, nm, k, temp, **kw)
    del lg
    if ws is None:
        rows_capacity = R
        nbytes = o.logits_fused_workspace_bytes(R, V, e.shape[1], k)
        assert nbytes > 0
        ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
        status = torch.zeros((2,), dtype=torch.int32, device="cuda")
    o.logits_fused(e, w, mp, ids_b, sc_b, nm, k, temp, ws, status, rows_capacity=rows_capacity, **kw)
    torch.cuda.synchronize()
    return ids_a, sc_a, ids_b, sc_b, status


def _units():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("R,V,b", [(300, 65536, 1), (64, 65536, 2), (2048, 65536, 8), (128 * 67, 65536, 67), (700, 8192, 7), (96, 1024, 3), (260, 4096, 2)])
@pytest.mark.parametrize("temp", [1.0, 0.0])
def test_fused_equals_materialised_philox(R, V, b, temp):
    """libmmg Philox keying: identical sampled tokens; scores equal to 2e-6 (the fused path sums the softmax denominator per list segment)."""
    e, w, b, n, nm, mp = _case(R, V, 512 if V == 65536 else 128, seed=R + V, b=b)
    k = math.ceil(0.1 * V)
    ids_a, sc_a, ids_b, sc_b, status = _run_both(e, w, b, n, nm, mp, k, temp, seed=1234, step=3, row_offset=5 * n)
    assert torch.equal(ids_a, ids_b), int((ids_a != ids_b).sum())
    assert float((sc_a - sc_b).abs().max()) < 2e-6
    assert int(status[1]) == 0
    print(f"R={R} V={V}: fallback rows {int(status[0])}")


def test_fused_equals_materialised_injected_noise_and_aten():
    e, w, b, n, nm, mp = _case(240, 8192, 128, seed=7, b=4)
    k = math.ceil(0.1 * 8192)
    u = torch.rand((b, n, 8192), device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    ids_a, sc_a, ids_b, sc_b, status = _run_both(e, w, b, n, nm, mp, k, 0.7, u=u)
    assert torch.equal(ids_a, ids_b) and float((sc_a - sc_b).abs().max()) < 2e-6
    off = torch.tensor([8], dtype=torch.int64, device="cuda"); seed_dev = torch.tensor([99], dtype=torch.int64, device="cuda")
    ids_a, sc_a, ids_b, sc_b, status = _run_both(e, w, b, n, nm, mp, k, 0.7, seed=0, seed_dev=seed_dev, aten=(16, off, 256 * 40))
    assert torch.equal(ids_a, ids_b) and float((sc_a - sc_b).abs().max()) < 2e-6


def test_fused_other_k_and_unsupported_shapes():
    """top-k thresholds other than 0.9; shapes the fused path declines (the caller then uses the materialised path)."""
    e, w, b, n, nm, mp = _case(256, 65536, 512, seed=11, b=2)
    o = ops()
    V = 65536
    for k in (math.ceil(0.05 * V), math.ceil(0.08 * V)):
        assert o.logits_fused_workspace_bytes(256, V, 512, k) > 0
        ids_a, sc_a, ids_b, sc_b, status = _run_both(e, w, b, n, nm, mp, k, 0.9, seed=5, step=1)
        assert torch.equal(ids_a, ids_b) and float((sc_a - sc_b).abs().max()) < 2e-6 and int(status[1]) == 0
    assert o.logits_fused_workspace_bytes(256, V, 512, math.ceil(0.2 * V)) == 0          # candidate lists would not fit: materialised path only
    assert o.logits_fused_workspace_bytes(256, 1000, 512, 100) == 0 and o.logits_fused_workspace_bytes(256, V, 100, 6554) == 0


def test_fused_fallback_rows_and_overflow_word():
    """Rows with constant logits (zero embedding): every logit ties, the candidate lists overflow, the row is redone from materialised logits
    inside the call (top-k keeps the lowest indices among equals -> same token as the materialised kernel).  More than 128 such rows in one
    call raise status[1]."""
    e, w, b, n, nm, mp = _case(384, 65536, 512, seed=13, b=3)
    k = math.ceil(0.1 * 65536)
    e[5] = 0; e[200] = 0; e[383] = 0
    ids_a, sc_a, ids_b, sc_b, status = _run_both(e, w, b, n, nm, mp, k, 1.0, seed=77, step=2)
    assert torch.equal(ids_a, ids_b) and float((sc_a - sc_b).abs().max()) < 2e-6
    assert int(status[0]) >= 3 and int(status[1]) == 0
    e[:200] = 0
    *_, status = _run_both(e, w, b, n, nm, mp, k, 1.0, seed=77, step=2)
    assert int(status[1]) == 1 and int(status[0]) >= 200


def test_generate_fused_tail_equals_materialised_and_overflow_rerun():
    """MaskGit.generate(): the fused tail (default) and the materialised tail give the same tokens and pixels, eager and under the CUDA graph;
    a model whose logits are constant (zero to_logits) overflows the fallback and is transparently re-run on the materialised path."""
    import muse_maskgit_pytorch_b200 as M
    from muse_maskgit_pytorch_b200 import t5
    t5.T5_CONFIGS["synth-128"] = {"d_model": 128}

    def build():
        tr = M.MaskGitTransformer(num_tokens=1024, dim=128, seq_len=16, depth=2, heads=2, t5_name="synth-128", precision="bf16")
        sd = util.transformer_sd(1024, 128, 16, 2, 2, seed=13, text_dim=128)
        full = tr.state_dict(); full.update(sd); tr.load_state_dict(full)
        vae = M.VQGanVAE(dim=16, layers=2, codebook_size=1024, precision="bf16")
        full = vae.state_dict(); full.update(util.vae_sd(16, 2, 1024, seed=12)); vae.load_state_dict(full)
        return M.MaskGit(image_size=16, transformer=tr.cuda(), vae=vae.cuda()).cuda()
    mg = build()
    te = util.text_embeds("g4.te", 3, 8, 128, 14).cuda()
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    mg.sampler_seed = 42
    outs = {}
    for fused in (True, False):
        for graph in (False, True):
            mg.use_fused_tail, mg.use_cuda_graph = fused, graph
            outs[(fused, graph)] = mg.generate(["a"] * 3, timesteps=8, return_ids=True)
    ref_img, ref_ids = outs[(False, False)]
    for key, (img, ids) in outs.items():
        assert torch.equal(ids, ref_ids), key
        assert float((img - ref_img).abs().max()) < 1e-6, key
    assert mg.last_fused_fallback_rows >= 0
    # degenerate model at V = 65536: all logits equal -> every row's lists overflow -> more fallback rows than the call holds -> overflow word
    # -> generate() repeats the call on the materialised path (same tokens as asking for that path directly)
    mg2, b_big = _degenerate_maskgit()
    mg2.sampler_seed = 42
    mg2.use_fused_tail = True
    img_f, ids_f = mg2.generate(["a"] * b_big, timesteps=4, return_ids=True)
    mg2.use_fused_tail = False
    img_m, ids_m = mg2.generate(["a"] * b_big, timesteps=4, return_ids=True)
    assert torch.equal(ids_f, ids_m) and torch.equal(img_f, img_m)


def _degenerate_maskgit():
    """V = 65536 model whose to_logits is zero: every logit of every row ties, so every sampled row takes the fallback and the first step
    of a 16-sequence batch (16 x 16 = 256 rows) has more of them than one fused call holds."""
    import muse_maskgit_pytorch_b200 as M
    from muse_maskgit_pytorch_b200 import t5
    t5.T5_CONFIGS["synth-128"] = {"d_model": 128}
    torch.manual_seed(5)
    tr = M.MaskGitTransformer(num_tokens=65536, dim=128, seq_len=16, depth=1, heads=2, t5_name="synth-128", precision="bf16")
    with torch.no_grad():
        tr.to_logits.weight.zero_()
    vae = M.VQGanVAE(dim=16, layers=2, codebook_size=65536, precision="bf16")
    mg = M.MaskGit(image_size=16, transformer=tr.cuda(), vae=vae.cuda()).cuda()
    te = util.text_embeds("g4.te", 3, 8, 128, 14).cuda().repeat(6, 1, 1)
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    return mg, 16


def test_generate_overflow_rerun_reuses_the_drawn_seed():
    """Without sampler_seed, generate() draws its sampling seed from torch's global generator once.  When the fused tail overflows, the
    materialised rerun uses that same seed: the tokens equal those of asking for the materialised path directly under the same
    manual_seed, and the generator has advanced by exactly one draw either way."""
    mg, b = _degenerate_maskgit()
    mg.sampler_seed = None
    torch.manual_seed(11)
    torch.randint(0, 2 ** 62, (1,))
    one_draw = torch.get_rng_state()
    outs = {}
    for fused in (True, False):
        mg.use_fused_tail = fused
        mg.last_fused_fallback_rows = 0
        torch.manual_seed(11)
        outs[fused] = mg.generate(["a"] * b, timesteps=4, return_ids=True)
        assert torch.equal(torch.get_rng_state(), one_draw), f"use_fused_tail={fused}: the global generator moved by more than one draw"
        if fused:
            assert mg.last_fused_fallback_rows > 128            # the fused attempt did overflow and was repeated
    assert torch.equal(outs[True][1], outs[False][1]) and torch.equal(outs[True][0], outs[False][0])


# ------------------------------------------------------------------------------------------------ split plans against an fp64 oracle
def _fp64_check(e, w, pos, ids, scores, rows, k, temp, u_rows, min_margin):
    """fp64 oracle (logits e . w^T from the same bf16 values) on `rows`: ids equal wherever the perturbed top-2 margin exceeds
    `min_margin` (at least 90 % of the rows), scores 1 - softmax[token] within 1e-5 there."""
    lg = (e[rows].double() @ w.double().T).cpu()
    pred, osc, margin = util.oracle_rows(lg, u_rows, temp, k)
    got, gsc = ids[pos].cpu(), scores[pos].cpu().double()
    ok = margin > min_margin
    assert float(ok.double().mean()) >= 0.9, f"only {int(ok.sum())} of {len(rows)} rows have a clear margin"
    bad = ok & (got != pred)
    assert not bad.any(), f"rows {[rows[i] for i in bad.nonzero().flatten().tolist()]}: got {got[bad].tolist()} want {pred[bad].tolist()}"
    err = float((gsc - osc)[ok].abs().max())
    assert err < 1e-5, err
    return int(ok.sum())


# (V, K, S, lowest row count): S = 1 and 2 are the plans whose finisher shares one list segment among 4 / 2 warps; the largest S has the
# shortest segments; V = 1280 has only S <= 2; V = 12288 samples every 3rd vocabulary row.  Every R is 77 rows past a multiple of 128.
PLANS = [(65536, 512, 1, 1), (65536, 512, 2, 1), (65536, 512, 64, 3000), (1024, 64, 1, 1), (1024, 64, 2, 1), (1024, 64, 4, 1000),
         (1280, 512, 2, 300), (12288, 1024, 8, 1)]


@pytest.mark.parametrize("V,K,S,lo", PLANS)
def test_fused_split_plans_vs_materialised_and_fp64_oracle(V, K, S, lo):
    """The row count is chosen on the card at hand (oracle/fused_tail.py restates the planner) so that the call runs with S splits of the
    vocabulary.  All rows equal the materialised path; one row per M-tile and every row of the ragged last tile equal the fp64 oracle on
    libmmg's Philox stream."""
    units = _units()
    R = FT.rows_for_plan(V, S, units, lo=lo)
    assert R is not None, f"no row count <= 40000 reaches S={S} at V={V} on {units} SMs"
    pl = FT.lf_plan(R, V, units)
    e, w, b, n, nm, mp = _case(R, V, K, seed=R + V + K)
    k = math.ceil(0.1 * V)
    seed, step, off = 1234, 3, 5 * n
    ids_a, sc_a, ids_b, sc_b, status = _run_both(e, w, b, n, nm, mp, k, 1.0, seed=seed, step=step, row_offset=off)
    assert torch.equal(ids_a, ids_b), int((ids_a != ids_b).sum())
    assert float((sc_a - sc_b).abs().max()) < 2e-6
    assert int(status[1]) == 0
    g = torch.Generator().manual_seed(R)
    tiles = pl["num_m_tiles"]
    rows = sorted(set((torch.arange(tiles - 1) * 128 + torch.randint(0, 128, (tiles - 1,), generator=g)).tolist()) | set(range((tiles - 1) * 128, R)))
    pos = mp[0].long().cpu()[rows]
    u = torch.stack([torch.from_numpy(philox.uniform(seed, step, off + int(p), V)) for p in pos])
    checked = _fp64_check(e, w, (0, pos), ids_b, sc_b, rows, k, 1.0, u, 1e-3)
    print(f"plan R={R} V={V} K={K} S={pl['S']} cap={pl['cap']} on {units} SMs: fallback rows {int(status[0])}, "
          f"fp64 oracle on {checked} of {len(rows)} rows")
    assert pl["S"] == S
    del ids_a, sc_a, ids_b, sc_b, e, w
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ constructed rows, exact logits
def _bf(x):
    return torch.as_tensor(x, dtype=torch.float32).to(bf).float()


def _constructed_rows(V, k, plan, g):
    """One logits row per case, as exactly representable bf16 values, and its injected uniforms.  Returns (names, logits [R, V] fp32,
    u [R, V]).  The cases and the leg each is built for:
      plain       random row                                                            candidate lists
      tie         8 logits equal to the k-th value but outside the top k get the largest noise (the lowest indices among equals are kept):
                  8 exclusions, then the last tie inside the top k wins                  candidate lists
      segment     every 3rd column of one (split, half) segment high, the rest of it low: 21-22 candidates per 64-column chunk,
                  more than the segment's list capacity                                   fallback
      fifo        31 candidates in each of 4 consecutive chunks of one segment (the entries left over from the chunk before plus 31 exceed
                  the 32 FIFO slots), the rest of the segment low: fewer than its capacity fallback
      threshold   the sampled columns (v % stride == 0) high, the rest low: fewer than k candidates                fallback
      excl10      the 10 logits ranked k .. k+9 get the largest noise: 10 exclusions    candidate lists
      excl30      the same with 30: more than the finisher's 24 exclusions               fallback"""
    npt, stride = plan["npt"], plan["stride"]
    names = ["plain", "tie", "segment", "fifo", "threshold", "excl10", "excl30"]
    x = _bf(torch.randn((len(names), V), generator=g))
    u = torch.rand((len(names), V), generator=g)
    hi = lambda m: _bf(5.0 + 0.5 * torch.randn((m,), generator=g))
    lo = lambda m: _bf(-5.0 + 0.5 * torch.randn((m,), generator=g))
    chunk = lambda sp, j, half: (sp * npt + j) * 128 + half * 64           # first column of chunk `half` of tile j of split sp

    def rank_order(row):
        return torch.argsort(-row.double(), stable=True)                    # by logit descending, ties by lowest index

    # tie: the members of the k-th value's tie group just past the top k (and the two last inside it) get increasing large noise
    r = names.index("tie")
    order = rank_order(x[r])
    c = x[r, order[k - 1]]
    ties = torch.nonzero(x[r] == c).flatten()                               # ascending index
    a = int((ties <= order[k - 1]).sum())                                   # tie members inside the top k
    assert len(ties) - a >= 8, "tie group too small"
    u[r] = 0.5 * u[r]
    sel = ties[max(a - 2, 0):a + 8]
    u[r, sel] = torch.linspace(0.98, 0.999, len(sel))
    # segment: split 2, half 0
    r = names.index("segment")
    for j in range(npt):
        c0 = chunk(2, j, 0)
        cols = torch.arange(c0, c0 + 64)
        high = cols % 3 == 0
        x[r, cols[high]] = hi(int(high.sum())); x[r, cols[~high]] = lo(int((~high).sum()))
    # fifo: split 1, half 0
    r = names.index("fifo")
    for j in range(npt):
        c0 = chunk(1, j, 0)
        x[r, c0:c0 + 64] = lo(64)
        if j < 4:
            x[r, c0:c0 + 31] = hi(31)
    # threshold miss
    r = names.index("threshold")
    smp = torch.arange(V) % stride == 0
    x[r, smp] = hi(int(smp.sum())); x[r, ~smp] = lo(int((~smp).sum()))
    # exclusion loop
    for name, m in (("excl10", 10), ("excl30", 30)):
        r = names.index(name)
        u[r] = 0.5 * u[r]
        u[r, rank_order(x[r])[k:k + m]] = torch.linspace(0.98, 0.999, m)
    return names, x, u


FALLBACK = {"plain": False, "tie": False, "segment": True, "fifo": True, "threshold": True, "excl10": False, "excl30": True}
BUILT_LEG = {"segment": "segment", "fifo": "fifo", "threshold": "threshold"}


def test_fused_constructed_rows_reach_their_leg_and_match_fp64_oracle():
    """One-hot embeddings: row r of e is the r-th unit vector, so logit[r, v] = w[v, r] exactly and each row's logits are built by hand
    (injected noise).  Every row equals the fp64 oracle; the rows built to fall back raise status[0] (one call per row, status never reset)
    and the others leave it unchanged; the rows through the lists agree with the host restatement of the candidate thresholds.  The same
    rows through the materialised sampler (mmg_logits_sample, no exclusion cap) equal the oracle too."""
    o = ops()
    V, K, temp = 65536, 512, 1.0
    k = math.ceil(0.1 * V)
    plan = FT.lf_plan(1, V, _units())
    names, x, u = _constructed_rows(V, k, plan, torch.Generator().manual_seed(17))
    R = len(names)
    assert FT.lf_plan(R, V, _units()) == plan
    # the construction: the host restatement sends each row down the leg it was built for
    gumbel = O.gumbel_from_uniform(u).numpy()
    for r, name in enumerate(names):
        leg = FT.fused_leg(x[r].numpy(), V, k, plan)
        assert leg == BUILT_LEG.get(name, "lists"), (name, leg)
        if leg == "lists":
            tok, passes = FT.fused_choice(x[r].numpy(), gumbel[r], k, temp, FT.sampled_threshold(x[r].numpy(), V, k))
            assert (tok is None) == FALLBACK[name], (name, passes)
    pred, osc, margin = util.oracle_rows(x.double(), u, temp, k)
    assert float(margin.min()) > 1e-4, margin.tolist()              # the noise leaves no near-tie: the ids must be exactly the oracle's
    w = torch.zeros((V, K), dtype=bf)
    w[:, :R] = x.T.to(bf)
    w = w.cuda()
    e = torch.zeros((R, K), dtype=bf, device="cuda")
    e[torch.arange(R), torch.arange(R)] = 1
    uc = u.cuda().view(R, 1, V)
    mp = torch.zeros((R, 1), dtype=torch.int32, device="cuda")
    nbytes = o.logits_fused_workspace_bytes(R, V, K, k)
    ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
    status = torch.zeros((2,), dtype=torch.int32, device="cuda")
    ids = torch.full((R, 1), V, dtype=torch.long, device="cuda"); sc = torch.full((R, 1), -1e5, device="cuda")
    o.logits_fused(e, w, mp, ids, sc, 1, k, temp, ws, status, rows_capacity=R, u=uc)        # all rows in one call
    st = status.tolist()
    assert st == [sum(FALLBACK.values()), 0], st
    assert torch.equal(ids[:, 0].cpu(), pred), (ids[:, 0].tolist(), pred.tolist())
    assert float((sc[:, 0].cpu().double() - osc).abs().max()) < 1e-5
    for r, name in enumerate(names):                                 # one row per call: which rows fell back
        idr = torch.full((1, 1), V, dtype=torch.long, device="cuda"); scr = torch.full((1, 1), -1e5, device="cuda")
        before = int(status[0])
        o.logits_fused(e[r:r + 1], w, mp[:1], idr, scr, 1, k, temp, ws, status, rows_capacity=R, u=uc[r:r + 1])
        fell = int(status[0]) - before
        print(f"constructed row {name}: fallback rows +{fell}")
        assert fell == int(FALLBACK[name]), (name, fell)
        assert int(idr) == int(pred[r]) and int(status[1]) == 0, name
    lg = torch.empty((R, V), device="cuda")
    o.linear(e, w, lg)
    assert torch.equal(lg.cpu(), x)                                  # one-hot rows: the logits are exact
    ids_m = torch.full((R, 1), V, dtype=torch.long, device="cuda"); sc_m = torch.full((R, 1), -1e5, device="cuda")
    o.logits_sample(lg, mp, ids_m, sc_m, 1, k, temp, u=uc)
    assert torch.equal(ids_m[:, 0].cpu(), pred), (ids_m[:, 0].tolist(), pred.tolist())
    assert float((sc_m[:, 0].cpu().double() - osc).abs().max()) < 1e-5


# ------------------------------------------------------------------------------------------------ one workspace across a mask schedule
def test_fused_workspace_reuse_across_decreasing_rows():
    """As generate() does: one workspace sized for the largest step and one status word that is never reset, then calls with fewer rows
    step after step (different split plans).  Every call equals the materialised path, nothing is written past the workspace, and a call
    with more rows than the capacity is refused before it launches anything."""
    from muse_maskgit_pytorch_b200 import _lib
    o = ops()
    V, K, R_cap = 65536, 512, 4173
    k = math.ceil(0.1 * V)
    nbytes = o.logits_fused_workspace_bytes(R_cap, V, K, k)
    guard = 1 << 16
    full = torch.full((nbytes + guard,), 0xA5, dtype=torch.uint8, device="cuda")
    ws, status = full[:nbytes], torch.zeros((2,), dtype=torch.int32, device="cuda")
    plans = []
    for R in (R_cap, 3500, 2817, 2100, 1500, 1000, 600, 300, 129, 77, 1):
        e, w, b, n, nm, mp = _case(R, V, K, seed=R)
        ids_a, sc_a, ids_b, sc_b, _ = _run_both(e, w, b, n, nm, mp, k, 1.0, ws=ws, status=status, rows_capacity=R_cap,
                                                seed=99, step=R % 7, row_offset=R)
        assert torch.equal(ids_a, ids_b), (R, int((ids_a != ids_b).sum()))
        assert float((sc_a - sc_b).abs().max()) < 2e-6, R
        assert int(status[1]) == 0, R
        plans.append(FT.lf_plan(R, V, _units())["S"])
    print(f"workspace reuse: S per step {plans}, fallback rows {int(status[0])}")
    assert len(set(plans)) > 1
    assert bool((full[nbytes:] == 0xA5).all()), "write past the workspace"
    e, w, b, n, nm, mp = _case(R_cap + 1, V, K, seed=5)
    ids = torch.full((b, n), V, dtype=torch.long, device="cuda"); sc = torch.full((b, n), -1e5, device="cuda")
    launches = _lib.launch_count()
    with pytest.raises(_lib.MMGError, match="rows_capacity"):
        o.logits_fused(e, w, mp, ids, sc, nm, k, 1.0, ws, status, rows_capacity=R_cap, seed=99)
    torch.cuda.synchronize()
    assert _lib.launch_count() == launches
    assert bool((ids == V).all()) and bool((sc == -1e5).all())


# ------------------------------------------------------------------------------------------------ only_masked (can_remask_prev_masked)
@pytest.mark.parametrize("sampler", ["fused", "materialised"])
def test_only_masked_writes_ids_of_masked_positions_only(sampler):
    """generate(can_remask_prev_masked=True) samples every position and keeps the decoded tokens: ids change only where they equalled
    mask_id (to the oracle's token), scores are written everywhere."""
    o = ops()
    V, K, b, n = 65536, 512, 4, 96
    k = math.ceil(0.1 * V)
    e, w, *_ = _case(b * n, V, K, seed=23)
    g = torch.Generator().manual_seed(23)
    ids0 = torch.randint(0, V, (b, n), generator=g)
    ids0[torch.rand((b, n), generator=g) < 0.5] = V                   # mask_id = V
    u = torch.rand((b, n, V), generator=g)
    mp = torch.arange(n, dtype=torch.int32).repeat(b, 1).cuda()
    ids = ids0.cuda(); sc = torch.full((b, n), -1e5, device="cuda")
    if sampler == "fused":
        nbytes = o.logits_fused_workspace_bytes(b * n, V, K, k)
        ws = torch.empty((nbytes,), dtype=torch.uint8, device="cuda"); status = torch.zeros((2,), dtype=torch.int32, device="cuda")
        o.logits_fused(e, w, mp, ids, sc, n, k, 0.8, ws, status, u=u.cuda(), only_masked_id=V)
        assert int(status[1]) == 0
    else:
        lg = torch.empty((b * n, V), device="cuda")
        o.linear(e, w, lg)
        o.logits_sample(lg, mp, ids, sc, n, k, 0.8, u=u.cuda(), only_masked_id=V)
    ids, sc = ids.cpu(), sc.cpu()
    masked = ids0 == V
    assert torch.equal(ids[~masked], ids0[~masked])
    assert bool((ids[masked] < V).all())
    assert bool((sc > -1e4).all())
    lg = (e.double() @ w.double().T).cpu()
    pred, osc, margin = util.oracle_rows(lg, u.view(b * n, V), 0.8, k)
    pred, osc, margin = pred.view(b, n), osc.view(b, n), margin.view(b, n)
    ok = margin > 1e-4
    assert float(ok.double().mean()) >= 0.9
    assert torch.equal(ids[masked & ok], pred[masked & ok])
    assert float((sc.double() - osc)[ok].abs().max()) < 1e-5


# ------------------------------------------------------------------------------------------------ the other finisher build
_MINB_CHILD = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
from muse_maskgit_pytorch_b200 import ops
d = torch.load(sys.argv[2])
e, w, mp = d["e"].cuda(), d["w"].cuda(), d["mp"].cuda()
ids = torch.full(d["ids_shape"], d["V"], dtype=torch.long, device="cuda"); sc = torch.full(d["ids_shape"], -1e5, device="cuda")
ws = torch.empty((ops.logits_fused_workspace_bytes(e.shape[0], d["V"], e.shape[1], d["k"]),), dtype=torch.uint8, device="cuda")
status = torch.zeros((2,), dtype=torch.int32, device="cuda")
ops.logits_fused(e, w, mp, ids, sc, d["nm"], d["k"], 1.0, ws, status, seed=1234, step=3)
torch.save(dict(ids=ids.cpu(), sc=sc.cpu(), status=status.cpu()), sys.argv[3])
"""


def test_finisher_minb6_build_equals_default(tmp_path):
    """MMG_FINISH_MINB=6 (read once per process) selects the finisher built for 6 CTAs per SM, which re-derives the Philox round keys
    per candidate: its ids and scores are bitwise those of the default build."""
    V, K = 65536, 512
    k = math.ceil(0.1 * V)
    e, w, b, n, nm, mp = _case(600, V, K, seed=29, b=3)
    torch.save(dict(e=e.cpu(), w=w.cpu(), mp=mp.cpu(), ids_shape=(b, n), V=V, nm=nm, k=k), tmp_path / "in.pt")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, MMG_FINISH_MINB="6")
    r = subprocess.run([sys.executable, "-c", _MINB_CHILD, root, str(tmp_path / "in.pt"), str(tmp_path / "out.pt")], env=env, cwd=root,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    got = torch.load(tmp_path / "out.pt")
    assert os.environ.get("MMG_FINISH_MINB", "4") == "4"
    ids_a, sc_a, ids_b, sc_b, status = _run_both(e, w, b, n, nm, mp, k, 1.0, seed=1234, step=3)
    assert torch.equal(got["ids"], ids_b.cpu()) and torch.equal(got["sc"], sc_b.cpu()) and torch.equal(got["status"], status.cpu())
    assert torch.equal(ids_a, ids_b)
