"""CPU: the host side of per-image sampling settings — argument checks, the fp32 tables the kernels read (bitwise the
values a scalar call hands them), and generate_sharded's slicing of per-image settings over two gloo ranks."""
import ctypes
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from muse_maskgit_pytorch_b200 import parallel


def _cpu_maskgit():
    import muse_maskgit_pytorch_b200 as M
    from muse_maskgit_pytorch_b200 import t5
    t5.T5_CONFIGS["synth-128"] = {"d_model": 128}
    tr = M.MaskGitTransformer(num_tokens=1024, dim=128, seq_len=16, depth=1, heads=2, t5_name="synth-128")
    return M.MaskGit(image_size=16, transformer=tr, vae=M.VQGanVAE(dim=16, layers=2, codebook_size=1024))


BAD = [dict(cond_scale=[3, 3]), dict(temperature=[1.0] * 4), dict(cond_scale=torch.ones(3, 1)), dict(cond_scale=[3, float("nan"), 3]),
       dict(temperature=float("inf")), dict(critic_noise_scale=[1, 1, float("-inf")]), dict(temperature=[1, -0.5, 1]),
       dict(temperature=-1), dict(cond_scale="3")]


@pytest.mark.parametrize("bad", BAD, ids=[str(i) for i in range(len(BAD))])
def test_bad_settings_raise_value_error(bad):
    """Checked on the host, so a model that never left the CPU raises them (test_gpu_batch_settings.py checks no launch happens)."""
    mg = _cpu_maskgit()
    images = torch.zeros((3, 3, 16, 16))
    for call in (lambda: mg.generate(["a"] * 3, **bad), lambda: mg.inpaint(["a"] * 3, images, torch.ones((3, 4, 4), dtype=torch.bool), **bad),
                 lambda: mg.edit(["a"] * 3, images, **bad)):
        with pytest.raises(ValueError):
            call()


def test_settings_tables_hold_the_scalar_call_values():
    """A uniform call's tables hold, bit for bit, the fp32 value each kernel argument had in a scalar call (ctypes rounds the same float64
    expression once); per-image values give each image its own column."""
    from muse_maskgit_pytorch_b200.muse_maskgit import _DecodeRequest, _per_image
    f32 = lambda v: ctypes.c_float(v).value
    T, b, n = 7, 3, 5
    for temperature, cond_scale, noise in ((1, 3, 1), (0.7, 1, 0.3), ([0.1, 1.7, 0.0], (1, 2.5, 7), torch.tensor([0.2, 0.0, 3.0]))):
        req = _DecodeRequest(texts=["a"] * b, cond_images=None, fmap_size=2, temperature=_per_image("t", temperature, b), topk_filter_thres=0.9,
                             timesteps=T, cond_scale=_per_image("c", cond_scale, b), critic_noise_scale=_per_image("n", noise, b),
                             can_remask_prev_masked=False, use_critic=True, return_ids=False)
        tab = req.settings(n)
        assert tab["temps"].shape == (T, b) and tab["crit_noise"].shape == (T, b * n) and tab["crit_cond_scale"].shape == (b * n,)
        for i in range(b):
            t_i = temperature if isinstance(temperature, (int, float)) else float(temperature[i])
            c_i = cond_scale if isinstance(cond_scale, (int, float)) else float(cond_scale[i])
            n_i = noise if isinstance(noise, (int, float)) else float(noise[i])
            for s, until in enumerate(reversed(range(T))):
                assert float(tab["temps"][s, i]) == f32(float(t_i * (until / T)))
                assert all(float(v) == f32(float(n_i * (until / T))) for v in tab["crit_noise"][s, i * n:(i + 1) * n])
            assert float(tab["cond_scale"][i]) == f32(float(c_i)) and bool((tab["crit_cond_scale"][i * n:(i + 1) * n] == f32(float(c_i))).all())
        assert req.branches == (1 if all(c == 1 for c in req.cond_scale) else 2)


class _StubMaskGit:
    class _T:
        encode_text = None

    class _V:
        channels = 3

    def __init__(self):
        self.transformer, self.row_offset, self.global_batch, self.sampler_seed = self._T(), 0, None, 7
        self.image_size, self.vae, self.seen = 4, self._V(), []

    def parameters(self):
        yield torch.zeros(1)

    def generate(self, texts, cond_images=None, **kw):
        self.seen.append(kw)
        return torch.full((len(texts), 3, 4, 4), float(self.row_offset))


def _worker(rank, world, port, total, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    mg = _StubMaskGit()
    scales = [float(i) for i in range(total)]
    parallel.generate_sharded(mg, ["t"] * total, cond_scale=scales, temperature=torch.arange(total, dtype=torch.float32) / 10,
                              critic_noise_scale=0.5, timesteps=3)
    lo, hi = parallel.shard_bounds(total, rank, world)
    kw = mg.seen[0] if mg.seen else None
    q.put((rank, lo, hi, None if kw is None else (list(kw["cond_scale"]), kw["temperature"].tolist(), kw["critic_noise_scale"], kw["timesteps"])))
    dist.barrier()
    dist.destroy_process_group()


def test_generate_sharded_slices_per_image_settings():
    total = 7
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, 29631, total, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    temps = (torch.arange(total, dtype=torch.float32) / 10).tolist()
    for rank, lo, hi, kw in got:
        assert kw == ([float(i) for i in range(lo, hi)], temps[lo:hi], 0.5, 3), (rank, kw)


def test_generate_sharded_rejects_a_wrong_length():
    with pytest.raises(ValueError):
        parallel.generate_sharded(_StubMaskGit(), ["t"] * 3, cond_scale=[1, 2])
