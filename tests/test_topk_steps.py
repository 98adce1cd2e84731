"""CPU: per-image `topk_filter_thres` and `timesteps`: parsing and its ValueErrors, the settings and count tables of a mixed request
(image b's column equals the column of a scalar request with its own (timesteps, threshold)), and, over gloo with two ranks, muse_sharded
forwarding each rank's slice of the new settings and every rank raising the same ValueError before any collective."""
import math

import pytest
import torch

from muse_maskgit_pytorch_b200 import parallel
from muse_maskgit_pytorch_b200.muse_maskgit import MaskGit, _DecodeRequest, _per_image, _per_image_steps


def test_steps_parsing():
    assert _per_image_steps(18, 3) == 18
    assert _per_image_steps([6, 6, 6], 3) == 6
    assert _per_image_steps((6, 4, 8), 3) == (6, 4, 8)
    assert _per_image_steps(torch.tensor([2, 5]), 2) == (2, 5)
    for bad in ([6, 0, 3], [6, 4], [6, 4.0, 2], [True, 2, 2], torch.tensor([1.0, 2.0, 3.0]), "abc"):
        with pytest.raises(ValueError):
            _per_image_steps(bad, 3)


def _req(T, thres, b=3, temps=(1.0, 0.5, 2.0), noise=(0.7, 0.2, 1.0)):
    return _DecodeRequest(texts=["a"] * b, cond_images=None, fmap_size=2, temperature=_per_image("t", list(temps), b), topk_filter_thres=thres,
                          timesteps=T, cond_scale=(3.0,) * b, critic_noise_scale=_per_image("n", list(noise), b),
                          can_remask_prev_masked=False, use_critic=True, return_ids=False)


def test_mixed_settings_columns_equal_scalar_requests():
    steps, thres, n, V = (6, 3, 8), (0.9, 0.95, 0.8), 4, 1024
    tab = _req(steps, thres).settings(n, V)
    assert tab["temps"].shape == (8, 3) and tab["crit_noise"].shape == (8, 12) and tab["k"].dtype == torch.int32
    for i, (T, th) in enumerate(zip(steps, thres)):
        one = _req(T, th).settings(n, V)
        assert torch.equal(tab["temps"][:T, i], one["temps"][:, i]) and bool((tab["temps"][T:, i] == 0).all())
        assert torch.equal(tab["crit_noise"][:T, i * n:(i + 1) * n], one["crit_noise"][:, i * n:(i + 1) * n])
        assert int(tab["k"][i]) == int(one["k"][i]) == math.ceil((1 - th) * V)


class _StubVae:
    channels = 3


def _stub_maskgit():
    mg = MaskGit.__new__(MaskGit)
    torch.nn.Module.__init__(mg)
    mg.noise_schedule = lambda t: torch.cos(t * math.pi * 0.5)
    mg.register_parameter("p", torch.nn.Parameter(torch.zeros(1)))
    return mg


def test_count_tables_and_rows():
    """Image b's column of the counts table is mask_schedule(N_b, T_b) then zeros; the rows of a step are its largest count, and with
    one timesteps they are mask_schedule(max N_b, T) as before."""
    mg = _stub_maskgit()
    counts, steps = [16, 5, 0, 16], (6, 3, 8, 2)
    r = mg._region(None, counts, steps, frozen=torch.zeros((4, 16), dtype=torch.uint8))
    tab = r.tensors["counts"]
    assert tab.shape == (8, 4) and "images" not in r.tensors
    for i, (c, T) in enumerate(zip(counts, steps)):
        want = (mg.mask_schedule(c, T) if c else [0] * T) + [0] * (8 - T)
        assert tab[:, i].tolist() == want
    assert list(r.rows) == [max(1, int(v)) for v in tab.max(dim=1).values]
    ru = mg._region(None, counts, 6, frozen=torch.zeros((4, 16), dtype=torch.uint8))
    assert list(ru.rows) == mg.mask_schedule(16, 6)
    assert list(mg._region(None, [0, 0], 4, frozen=torch.zeros((2, 16), dtype=torch.uint8)).rows) == mg.mask_schedule(0, 4)


def test_threshold_and_round_steps_validation():
    mg = _stub_maskgit()
    mg.transformer = type("T", (), {"num_tokens": 1024})()
    assert mg._thres_arg(0.9, 3) == 0.9
    assert mg._thres_arg([0.9, 0.5, 0.0], 3) == (0.9, 0.5, 0.0)
    for bad in ([0.9, 1.0, 0.9], [0.9, -0.5, 0.9], [0.9, 0.9], [0.9, float("nan"), 0.9]):
        with pytest.raises(ValueError):
            mg._thres_arg(bad, 3)
    mg.sampler_rng = "aten"
    with pytest.raises(ValueError, match="aten"):
        mg._steps_arg([6, 4, 4], 3)
    assert mg._steps_arg(6, 3) == 6 and mg._steps_arg([4, 4, 4], 3) == 4
    for method in ("edit", "extrapolate"):
        with pytest.raises(ValueError, match="step counter"):
            MaskGit._round_steps(method, [3, 3])
    MaskGit._round_steps("edit", 3)


class _StubMaskGit:
    """What parallel._run_shard reads of a MaskGit, with MaskGit's own argument checks; generate() / forward() record their kwargs."""
    _steps_arg, _thres_arg = MaskGit._steps_arg, MaskGit._thres_arg

    def __init__(self, rng="mmg"):
        self.transformer = type("T", (), {"num_tokens": 1024, "encode_text": None})()
        self.row_offset, self.global_batch, self.sampler_seed, self.sampler_rng, self.seen = 0, None, 7, rng, []

    def generate(self, texts, **kw):
        self.seen.append(kw)
        return torch.zeros((len(texts), 3, 4, 4))


class _StubMuse:
    def __init__(self, rng="mmg"):
        self.base_maskgit, self.superres_maskgit = _StubMaskGit(rng), _StubMaskGit()

    def forward(self, texts, **kw):
        self.base_maskgit.seen.append(kw)
        return torch.zeros((len(texts), 3, 8, 8)), torch.zeros((len(texts), 3, 4, 4))


def _raises(fn):
    try:
        fn()
    except ValueError:
        return True
    return False


def _gloo_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    texts = ["t"] * 4
    muse = _StubMuse()
    kw = dict(timesteps=[6, 4, 8, 2], superres_timesteps=(3, 4, 5, 6), cond_scale=[1.0, 2.0, 3.0, 4.0])
    hi, lo = parallel.muse_sharded(muse, texts, text_embeds=torch.zeros((4, 2, 3)), return_pil_images=False, return_lowres=True, **kw)
    seen = {k: list(v) for k, v in muse.base_maskgit.seen[0].items() if k in kw}
    # every rank raises before any collective: a rank that ran on would wait in the all-gather (and the test would time out)
    raised = [
        _raises(lambda: parallel.muse_sharded(_StubMuse("aten"), texts, timesteps=[6, 6, 4, 4], return_pil_images=False)),
        _raises(lambda: parallel.generate_sharded(_StubMaskGit("aten"), texts, timesteps=[6, 4, 6, 6])),
        _raises(lambda: parallel.generate_sharded(_StubMaskGit(), texts, topk_filter_thres=[0.9, 1.0, 0.9, 0.9])),
        _raises(lambda: parallel.generate_sharded(_StubMaskGit(), texts, timesteps=[6, 4, 0, 6])),
        _raises(lambda: parallel.edit_sharded(_StubMaskGit(), ["t"], torch.zeros((1, 3, 4, 4)), timesteps=[3])),   # rank 1 holds no row
    ]
    q.put((rank, seen, tuple(hi.shape), tuple(lo.shape), raised))
    dist.barrier()
    dist.destroy_process_group()


def test_muse_sharded_forwards_per_image_steps_and_every_rank_raises():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, 29731, q)) for r in range(2)]
    for p in procs:
        p.start()
    outs = dict((r, rest) for r, *rest in (q.get(timeout=180) for _ in range(2)))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, (seen, hi_shape, lo_shape, raised) in outs.items():
        lo_, hi_ = parallel.shard_bounds(4, rank, 2)
        assert seen == dict(timesteps=[6, 4, 8, 2][lo_:hi_], superres_timesteps=[3, 4, 5, 6][lo_:hi_], cond_scale=[1.0, 2.0, 3.0, 4.0][lo_:hi_])
        assert hi_shape == (4, 3, 8, 8) and lo_shape == (4, 3, 4, 4)
        assert all(raised), (rank, raised)
