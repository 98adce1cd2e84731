"""CPU, world_size 2 over gloo: the host-side sharding logic of the N>1 path (shard bounds, row offsets, one all-gather,
uneven shards).  The generate() call itself is replaced by a stub keyed on the global row — the CUDA path is covered by
the -m gpu tests (Philox shard invariance) and by bench.py --gpus N."""
import os
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from muse_maskgit_pytorch_b200 import parallel


class StubMaskGit:
    """generate() returns images that encode (global row, text embedding sum) so order and offsets are checkable."""
    class _T:
        encode_text = None
    class _V:
        channels = 3
    def __init__(self, seed=None):
        self.transformer, self.row_offset, self.global_batch, self.sampler_seed = self._T(), 0, None, seed
        self.image_size, self.vae, self.seen = 4, self._V(), []
    def parameters(self):
        yield torch.zeros(1)
    def generate(self, texts, cond_images=None, **kw):
        self.seen.append((self.sampler_seed, self.global_batch, self.row_offset))
        te = self.transformer.encode_text(texts)
        rows = torch.arange(self.row_offset, self.row_offset + len(texts), dtype=torch.float32)
        img = rows[:, None, None, None] * torch.ones((len(texts), 3, 4, 4)) + te.sum(dim=(1, 2))[:, None, None, None] * 1000
        if cond_images is not None:
            img = img + cond_images.mean(dim=(1, 2, 3))[:, None, None, None]
        return img


def _worker(rank, world, port, total, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    te = torch.arange(total * 6, dtype=torch.float32).view(total, 2, 3)
    cond = torch.arange(total, dtype=torch.float32).view(total, 1, 1, 1).expand(total, 3, 2, 2).contiguous()
    mg = StubMaskGit(seed=None if rank else 4242)       # rank 0's seed must reach every rank
    sentinel = mg.transformer.encode_text
    out = parallel.generate_sharded(mg, ["t"] * total, text_embeds=te, cond_images=cond, timesteps=3)
    # the call leaves the model as it found it (ADVICE r1: encode_text / row_offset / global_batch / seed were left overwritten)
    assert mg.transformer.encode_text is sentinel and mg.row_offset == 0 and mg.global_batch is None
    assert mg.sampler_seed == (None if rank else 4242)
    lo, hi = parallel.shard_bounds(total, rank, world)
    assert mg.seen == ([(4242, total, lo)] if hi > lo else []), mg.seen
    q.put((rank, out.numpy()))      # by value: a shared tensor's storage would be fetched from this process, which may have exited by then
    dist.barrier()
    dist.destroy_process_group()


def _run(total, port):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, total, q)) for r in range(2)]
    for p in procs:
        p.start()
    outs = {rank: torch.from_numpy(out) for rank, out in (q.get(timeout=120) for _ in range(2))}
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return outs


def test_shard_bounds():
    assert [parallel.shard_bounds(64, r, 8) for r in range(8)] == [(8 * r, 8 * r + 8) for r in range(8)]
    assert [parallel.shard_bounds(7, r, 2) for r in range(2)] == [(0, 4), (4, 7)]
    assert [parallel.shard_bounds(3, r, 4) for r in range(4)] == [(0, 1), (1, 2), (2, 3), (3, 3)]


def test_two_ranks_equal_single_rank_even_and_uneven():
    for total, port in ((8, 29611), (7, 29612), (1, 29613)):       # even, uneven, and an empty shard on rank 1
        outs = _run(total, port)
        te = torch.arange(total * 6, dtype=torch.float32).view(total, 2, 3)
        cond = torch.arange(total, dtype=torch.float32).view(total, 1, 1, 1).expand(total, 3, 2, 2).contiguous()
        single = StubMaskGit()
        single.transformer.encode_text = lambda t: te
        ref = single.generate(["t"] * total, cond_images=cond)
        assert torch.equal(outs[0], ref) and torch.equal(outs[1], ref)
