"""The fused logits kernel (tc_logits_kernel) runs its candidate / softmax epilogue straight from the wgmma accumulator fragments: each lane
of a quad gathers one (row, 64-column half) chunk with shuffles and runs the same per-chunk code as before.  What it writes is pinned
bit for bit:
  - every `parts` record and the written prefix of every list segment (min(ceil(count / 4) * 4, cap) entries), plus ids and scores, hash
    to what the staged-epilogue kernel wrote on the same seeded inputs (tests/golden/logits_fragment_epilogue.json, recorded on a
    132-SM H100 by running this module with --record);
  - each list segment of a row that stays on the lists is, entry for entry, the logits >= thr[row] of the materialised ops.linear product
    in column order;
  - every call stays on the fused path (status == [the constructed fallback rows, 0]);
  - a CUDA-graph replay writes the same bytes as the eager call.
The cases cover the S = 1, 2 and 64 split plans at V = 65536 (each with a ragged last M-tile), V = 1280 with an odd number of tiles per
split, and the hand-built rows whose 64-column chunks overflow the FIFO or whose segment overflows its list capacity."""
import hashlib
import json
import math
import os
import sys

import pytest
import torch

from oracle import fused_tail as FT

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
bf = torch.bfloat16
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "logits_fragment_epilogue.json")
CASES = ["S1", "S2", "S64", "V1280", "constructed"]


def ops():
    from muse_maskgit_pytorch_b200 import ops as _ops
    return _ops


def _units():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _up(x):
    return (x + 255) // 256 * 256


def _carve(R_max, V, units):
    """Byte offsets of thr, parts and lists in the workspace (mmg_logits_fused's lf_carve, restated)."""
    parts = lists = 0
    R = FT.LF_BM
    while True:
        Rc = min(R, R_max)
        pl = FT.lf_plan(Rc, V, units)
        parts = max(parts, Rc * pl["S"] * FT.LF_SEGS * 16)
        lists = max(lists, Rc * pl["S"] * FT.LF_SEGS * pl["cap"] * 8)
        if R >= R_max:
            break
        R += FT.LF_BM
    ns = FT.lf_plan(1, V, units)["ns"]
    thr = _up(R_max * ns * 4)
    o_parts = thr + _up(R_max * 4)
    return thr, o_parts, o_parts + _up(parts)


def _inputs(name, units):
    """(e, w, u or None, fallback rows from the finisher's exclusion cap) of a case, drawn on the host from fixed seeds."""
    if name == "constructed":
        from tests import test_gpu_fused_tail as FTT
        V, K = 65536, 512
        k = math.ceil(0.1 * V)
        plan = FT.lf_plan(1, V, units)
        names, x, u = FTT._constructed_rows(V, k, plan, torch.Generator().manual_seed(17))
        R = len(names)
        w = torch.zeros((V, K), dtype=bf)
        w[:, :R] = x.T.to(bf)
        e = torch.zeros((R, K), dtype=bf)
        e[torch.arange(R), torch.arange(R)] = 1
        # the rows built for the finisher's exclusion cap fall back on top of those the lists show (threshold, fifo, segment)
        return e.cuda(), w.cuda(), u.view(R, 1, V).cuda(), sum(FTT.FALLBACK[n] and n not in FTT.BUILT_LEG for n in names)
    V, K, S, lo = {"S1": (65536, 512, 1, 1), "S2": (65536, 512, 2, 1), "S64": (65536, 512, 64, 3000), "V1280": (1280, 512, 2, 300)}[name]
    R = FT.rows_for_plan(V, S, units, lo=lo)
    assert R is not None and R % FT.LF_BM == 77
    g = torch.Generator().manual_seed(R + V + S)
    e = torch.randn((R, K), generator=g).to(bf)
    w = (torch.randn((V, K), generator=g) * K ** -0.5).to(bf)
    return e.cuda(), w.cuda(), None, 0


class _Call:
    """One fused call on its own workspace: the bytes it writes (parts records, written list prefixes) and its ids / scores."""

    def __init__(self, e, w, u, units):
        o = ops()
        self.R, self.K = e.shape
        self.V = w.shape[0]
        self.k = math.ceil(0.1 * self.V)
        self.plan = FT.lf_plan(self.R, self.V, units)
        nm = 1 if u is not None else self.R
        self.b = self.R // nm
        self.ws = torch.zeros((o.logits_fused_workspace_bytes(self.R, self.V, self.K, self.k),), dtype=torch.uint8, device="cuda")
        self.status = torch.zeros((2,), dtype=torch.int32, device="cuda")
        self.mp = torch.arange(nm, dtype=torch.int32, device="cuda").repeat(self.b, 1).contiguous()
        self.ids = torch.full((self.b, nm), self.V, dtype=torch.long, device="cuda")
        self.sc = torch.full((self.b, nm), -1e5, device="cuda")
        self.args = (e, w, self.mp, self.ids, self.sc, nm, self.k, 1.0, self.ws, self.status)
        self.kw = dict(rows_capacity=self.R, u=u) if u is not None else dict(rows_capacity=self.R, seed=1234, step=3, row_offset=11)

    def run(self):
        ops().logits_fused(*self.args, **self.kw)

    def reset(self):
        self.ws.zero_(); self.status.zero_(); self.ids.fill_(self.V); self.sc.fill_(-1e5)

    def written(self, units):
        """parts [R, S, 2] as (max, sum, count, overflow) words, lists [R * S * 2, cap] x (logit bits, index), the written-prefix mask."""
        S, cap = self.plan["S"], self.plan["cap"]
        o_thr, o_parts, o_lists = _carve(self.R, self.V, units)
        nseg = self.R * S * FT.LF_SEGS
        parts = self.ws[o_parts:o_parts + nseg * 16].view(torch.int32).view(nseg, 4)
        lists = self.ws[o_lists:o_lists + nseg * cap * 8].view(torch.int32).view(nseg, cap, 2)
        thr = self.ws[o_thr:o_thr + self.R * 4].view(torch.float32)
        count = parts[:, 2].long()
        written = torch.clamp((count + 3) // 4 * 4, max=cap)
        mask = torch.arange(cap, device="cuda")[None, :] < written[:, None]
        return parts, lists, mask, thr

    def digest(self, units):
        parts, lists, mask, _ = self.written(units)
        h = hashlib.sha256(parts.cpu().numpy().tobytes())
        h.update(lists[mask].cpu().numpy().tobytes())
        return dict(ws_sha256=h.hexdigest(), ids_sha256=hashlib.sha256(self.ids.cpu().numpy().tobytes()).hexdigest(),
                    scores_sha256=hashlib.sha256(self.sc.cpu().numpy().tobytes()).hexdigest(), status=self.status.tolist(),
                    R=self.R, S=self.plan["S"])


def _record(path):
    units = _units()
    out = {"units": units, "device": torch.cuda.get_device_name(), "cases": {}}
    for name in CASES:
        e, w, u, _ = _inputs(name, units)
        c = _Call(e, w, u, units)
        c.run()
        torch.cuda.synchronize()
        out["cases"][name] = c.digest(units)
        if name == "constructed":
            out["cases"][name]["ids"] = c.ids.flatten().tolist()
            out["cases"][name]["scores"] = c.sc.flatten().tolist()
        print(name, out["cases"][name]["R"], out["cases"][name]["S"], out["cases"][name]["status"], flush=True)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)


def _lists_vs_materialised(c, e, w, units):
    """Segments of rows without overflow: the list entries are the logits >= thr[row] of the materialised product, in column order.
    Returns the rows the finisher must send to the fallback before its exclusion loop: fewer than k candidates, or an overflow."""
    S, npt, cap = c.plan["S"], c.plan["npt"], c.plan["cap"]
    parts, lists, _, thr = c.written(units)
    lg = torch.empty((c.R, c.V), device="cuda")
    ops().linear(e, w, lg)
    cols = torch.arange(c.V, device="cuda", dtype=torch.int32)
    seg_view = lambda t: t.view(-1, S, npt, FT.LF_SEGS, 64).transpose(2, 3).reshape(-1, npt * 64)     # [R * S * 2, npt * 64] in column order
    x = seg_view(lg)
    col = seg_view(cols.expand(c.R, c.V))
    cand = x >= thr.repeat_interleave(S * FT.LF_SEGS)[:, None]
    count = cand.sum(1)
    ovf = parts[:, 3] != 0
    assert torch.equal(count[~ovf], parts[~ovf, 2].long()), "candidate counts"
    pos = torch.cumsum(cand.int(), 1) - 1
    keep = cand & (pos < cap) & ~ovf[:, None]
    want = torch.zeros((x.shape[0], cap, 2), dtype=torch.int32, device="cuda")
    seg = torch.arange(x.shape[0], device="cuda")[:, None].expand_as(pos)
    want[seg[keep], pos[keep], 0] = x.view(torch.int32)[keep]
    want[seg[keep], pos[keep], 1] = col[keep]
    valid = (torch.arange(cap, device="cuda")[None, :] < count[:, None]) & ~ovf[:, None]
    assert torch.equal(lists[valid], want[valid]), "list entries differ from the materialised logits"
    row_short = count.view(c.R, -1).sum(1) < c.k
    row_ovf = ovf.view(c.R, -1).any(1)
    return int((row_short | row_ovf).sum())


@pytest.mark.parametrize("name", CASES)
def test_fragment_epilogue_bytes(name):
    units = _units()
    with open(GOLDEN) as f:
        G = json.load(f)
    e, w, u, excl_fallbacks = _inputs(name, units)
    c = _Call(e, w, u, units)
    c.run()
    torch.cuda.synchronize()
    d = c.digest(units)
    fallbacks = _lists_vs_materialised(c, e, w, units) + excl_fallbacks
    print(f"{name}: R={c.R} S={c.plan['S']} npt={c.plan['npt']} cap={c.plan['cap']}: status {c.status.tolist()}")
    assert c.status.tolist() == [fallbacks, 0], (c.status.tolist(), fallbacks)
    # a CUDA-graph replay writes the same bytes
    c.reset()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        c.run()                                                      # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c.run()
    c.reset()
    graph.replay()
    torch.cuda.synchronize()
    assert c.digest(units) == d, "CUDA-graph replay differs from the eager call"
    if G["units"] != units:
        pytest.skip(f"goldens recorded on {G['units']} SMs, this card has {units}: the split plans differ")
    g = G["cases"][name]
    assert (d["R"], d["S"]) == (g["R"], g["S"])
    assert d["status"] == g["status"]
    assert d["ws_sha256"] == g["ws_sha256"], "parts / lists bytes differ from the staged-epilogue kernel"
    assert d["ids_sha256"] == g["ids_sha256"] and d["scores_sha256"] == g["scores_sha256"], "ids / scores differ"
    if "ids" in g:
        assert c.ids.flatten().tolist() == g["ids"] and c.sc.flatten().tolist() == g["scores"]


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--record":
        _record(sys.argv[2])
    else:
        sys.exit("usage: python -m tests.test_gpu_logits_fragment_epilogue --record OUT.json")
