"""GPU: the launch sequence of the MaskGit decode path, pinned.

Every libmmg entry point that generate(), inpaint(), edit() and MaskGit.forward call is recorded in order, with the non-pointer fields
of its argument struct (nested structs included, floats as repr), for one scenario per decode-path branch: CFG on and off, eager and
whole-call graph (a replay adds no host launch), injected noise, re-masking of decoded tokens, both critics, self-conditioning, the
super-resolution model, fp8, the native decode step, ragged inpainting, editing, the fused tail's overflow rerun, the training loss and
the ATen noise stream.  The sequences must equal tests/golden/decode_launch_trace.json exactly: a change to how the decode loop is
orchestrated on the host may not change what runs on the device.

MMG_RECORD_TRACE=<path> records the fixture at <path> instead of comparing (one scenario per test, merged into the file)."""
import ctypes
import json
import os
import random

import pytest
import torch

from oracle import synth
from tests import util
from tests.test_gpu_fp8 import small_maskgit
from tests.test_gpu_fused_tail import _degenerate_maskgit
from tests.test_gpu_models import make_branch_maskgit, make_maskgit

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)
GOLDEN = os.path.join(util.GOLDEN, "decode_launch_trace.json")
RECORD = os.environ.get("MMG_RECORD_TRACE")


def _fields(st):
    out = []
    for name, typ in st._fields_:
        if typ is ctypes.c_void_p or issubclass(typ, ctypes._Pointer):
            continue
        v = getattr(st, name)
        if isinstance(v, ctypes.Structure):
            v = _fields(v)
        elif isinstance(v, float):
            v = repr(v)
        out.append([name, v])
    return out


def _te():
    return util.text_embeds("g4.te", 3, 8, 128, 14).cuda()


def _setup(mg, seed=7, graph=False, te=None):
    te = _te() if te is None else te
    mg.transformer.encode_text = lambda texts: te[:len(texts)]
    mg.sampler_seed, mg.use_cuda_graph = seed, graph
    return mg


def _images(b, size):
    return torch.from_numpy(synth.uniform("trace.img", (b, 3, size, size), 31)).cuda()


def _ragged(b, f, fracs, seed=1):
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.rand((f, f), generator=g) < fr if 0 < fr < 1 else torch.full((f, f), fr >= 1) for fr in fracs]).cuda()


# Each scenario builds its models (not recorded) and returns the calls whose launches are recorded, one list per call.
def _generate(cond_scale, graph):
    mg = _setup(make_maskgit("bf16"), graph=graph)
    run = lambda: mg.generate(["a"] * 3, timesteps=6, cond_scale=cond_scale)
    return [run, run]


def _injected():
    mg = _setup(make_maskgit("fp32"))
    mg.sampler_noise_fn = util.torch_noise_fn(777)
    return [lambda: mg.generate(["a"] * 3, timesteps=6)]


def _branch(name, graph=False):
    mg, kw, _ = make_branch_maskgit(name, "bf16")
    _setup(mg, graph=graph)
    run = lambda: mg.generate(["a"] * 3, timesteps=5, **kw)
    return [run, run] if graph else [run]


def _superres():
    mg = _setup(make_maskgit("bf16", superres=True))
    cond = _images(2, 16)
    return [lambda: mg.generate(["a"] * 2, cond_images=cond, timesteps=4)]


def _fp8(graph):
    mg = small_maskgit("fp8")
    mg.sampler_seed, mg.use_cuda_graph = 17, graph
    run = lambda: mg.generate(["a"] * 3, timesteps=4)
    return [run, run] if graph else [run]


def _native(graph):
    mg = _setup(make_maskgit("bf16"), graph=graph)
    mg.use_native_step = True
    run = lambda: mg.generate(["a"] * 3, timesteps=6)
    return [run, run] if graph else [run]


def _inpaint(graph):
    mg = _setup(make_maskgit("bf16"), graph=graph)
    img, m = _images(3, 16), _ragged(3, 4, [0.5, 1, 0])
    run = lambda: mg.inpaint(["a"] * 3, img, m, timesteps=6)
    return [run, run]


def _edit(graph, iterations):
    mg = _setup(make_maskgit("bf16"), graph=graph)
    img, m = _images(3, 16), _ragged(3, 4, [0.3, 1, 0.6])
    run = lambda: mg.edit(["a"] * 3, img, mask=m, iterations=iterations, fraction=0.5, timesteps=3)
    return [run, run]


def _overflow(kind):
    mg, b = _degenerate_maskgit()
    mg.sampler_seed, mg.use_cuda_graph = 42, False
    if kind == "generate":
        return [lambda: mg.generate(["a"] * b, timesteps=4)]
    img = _images(b, 16)
    m = torch.rand((b, 4, 4), generator=torch.Generator().manual_seed(7)) < 0.6
    m[0] = True
    return [lambda: mg.edit(["a"] * b, img, mask=m.cuda(), iterations=2, fraction=0.6, timesteps=3)]


def _forward(critic, rng="mmg"):
    mg, _, _ = make_branch_maskgit("gen_critic_small", "bf16") if critic else (make_maskgit("bf16"), None, None)
    mg.sampler_seed, mg.sampler_rng = 3, rng
    te = _te()
    ids = torch.randint(0, 1024, (3, 16), generator=torch.Generator().manual_seed(9)).cuda()

    def run():
        random.seed(4)
        return mg(ids, text_embeds=te)
    return [run]


def _aten():
    mg = _setup(make_maskgit("bf16"))
    mg.sampler_rng = "aten"
    return [lambda: mg.generate(["a"] * 3, timesteps=4)]


SCENARIOS = {
    "generate_cfg3_eager": lambda: _generate(3, False),
    "generate_cfg1_eager": lambda: _generate(1, False),
    "generate_cfg3_graph": lambda: _generate(3, True),
    "generate_cfg1_graph": lambda: _generate(1, True),
    "generate_injected_noise": _injected,
    "generate_remask_prev_masked": lambda: _branch("gen_remask_prev_small"),
    "generate_token_critic": lambda: _branch("gen_critic_small"),
    "generate_token_critic_graph": lambda: _branch("gen_critic_small", graph=True),
    "generate_self_token_critic": lambda: _branch("gen_selfcritic_small"),
    "generate_self_cond": lambda: _branch("gen_selfcond_small"),
    "generate_superres": _superres,
    "generate_fp8_eager": lambda: _fp8(False),
    "generate_fp8_graph": lambda: _fp8(True),
    "generate_native_step": lambda: _native(False),
    "generate_native_step_graph": lambda: _native(True),
    "inpaint_ragged_eager": lambda: _inpaint(False),
    "inpaint_ragged_graph": lambda: _inpaint(True),
    "edit_mask_eager": lambda: _edit(False, 2),
    "edit_mask_graph": lambda: _edit(True, 2),
    "edit_zero_iterations": lambda: _edit(False, 0),
    "overflow_rerun_generate": lambda: _overflow("generate"),
    "overflow_rerun_edit": lambda: _overflow("edit"),
    "forward": lambda: _forward(False),
    "forward_token_critic": lambda: _forward(True),
    "aten_generate": _aten,
    "aten_forward_token_critic": lambda: _forward(True, rng="aten"),
}
ATEN = {"aten_generate", "aten_forward_token_critic"}      # offsets follow ATen's launch geometry, which depends on the SM count


def _record(calls, monkeypatch):
    from muse_maskgit_pytorch_b200 import _lib
    real, segments = _lib.call, []

    def call(name, args, stream=None):
        segments[-1].append([name, _fields(args)])
        return real(name, args, stream)
    monkeypatch.setattr(_lib, "call", call)
    for fn in calls:
        segments.append([])
        fn()
    torch.cuda.synchronize()
    monkeypatch.setattr(_lib, "call", real)
    return segments


def _pack(segments):
    """One table of distinct (name, fields) launches per scenario and each call's launches as indices into it."""
    table, index = [], {}
    calls = []
    for seg in segments:
        idx = []
        for e in seg:
            k = json.dumps(e)
            if k not in index:
                index[k] = len(table)
                table.append(e)
            idx.append(index[k])
        calls.append(idx)
    return dict(table=table, calls=calls)


def _unpack(s):
    return [[s["table"][i] for i in idx] for idx in s["calls"]]


@pytest.mark.parametrize("name", list(SCENARIOS))
def test_decode_launch_trace_matches_fixture(name, monkeypatch):
    torch.manual_seed(0)
    random.seed(0)
    props = torch.cuda.get_device_properties(0)
    calls = SCENARIOS[name]()
    torch.manual_seed(1)
    got = _record(calls, monkeypatch)
    if RECORD:
        data = json.load(open(RECORD)) if os.path.exists(RECORD) else dict(device=props.name, sm_count=props.multi_processor_count,
                                                                          scenarios={})
        data["scenarios"][name] = _pack(got)
        with open(RECORD, "w") as f:
            json.dump(data, f, separators=(",", ":"))
        return
    data = json.load(open(GOLDEN))
    if name in ATEN and props.multi_processor_count != data["sm_count"]:
        pytest.skip(f"recorded on {data['sm_count']} SMs ({data['device']}); this device has {props.multi_processor_count}")
    want = _unpack(data["scenarios"][name])
    assert [len(c) for c in got] == [len(c) for c in want], (name, [len(c) for c in got], [len(c) for c in want])
    for ci, (g, w) in enumerate(zip(got, want)):
        for li, (ge, we) in enumerate(zip(g, w)):
            assert ge == we, f"{name}: call {ci}, launch {li}: got {ge}, want {we}"
    if name.endswith("_graph"):
        assert got[1] == [], "a replay of the captured call launches nothing from the host"
