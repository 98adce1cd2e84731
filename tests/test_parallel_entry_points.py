"""CPU, gloo: the host side of the sharded entry points (generate_sharded with return_ids, inpaint_sharded, edit_sharded, muse_sharded)
over 2 and 3 spawned ranks with even, uneven and empty shards.  The model calls are stubs whose outputs encode the global row, the seed
and every per-row input they were given, so a rank that saw the wrong rows, seed or offsets returns something else than the
single-process call.  The CUDA path is covered by tests/test_gpu_sharded_entry_points.py."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from muse_maskgit_pytorch_b200 import parallel
from muse_maskgit_pytorch_b200.muse_maskgit import Muse

SEED = 4242


class StubMaskGit:
    """generate / inpaint / edit return images whose first values are features of each row (global row, text embedding sum, input
    image mean, mask sum, conditioning image mean, per-image settings, seed) and ids filled with the global row; every call is recorded."""
    class _T:
        encode_text = None

    class _V:
        channels = 3

        def get_encoded_fmap_size(self, size):
            return size // 2

    def __init__(self, seed=None, image_size=4, fail=False):
        self.transformer, self.row_offset, self.global_batch, self.sampler_seed = self._T(), 0, None, seed
        self.image_size, self.vae, self.sampler_rng, self.fail, self.calls = image_size, self._V(), "mmg", fail, []

    def parameters(self):
        yield torch.zeros(1)

    def _call(self, name, texts, images=None, mask=None, cond_images=None, return_ids=False, **kw):
        b = len(texts)
        self.calls.append(dict(name=name, seed=self.sampler_seed, row_offset=self.row_offset, global_batch=self.global_batch,
                               images=None if images is None else images.numpy(), mask=None if mask is None else mask.numpy(),
                               cond_images=None if cond_images is None else cond_images.numpy(),
                               settings={k: (v.tolist() if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}))
        if self.fail:
            raise RuntimeError("stub failure")
        te = self.transformer.encode_text(texts)
        per_row = lambda v: torch.as_tensor(v, dtype=torch.float32).expand(b) if v is not None else torch.zeros(b)
        feats = [torch.arange(self.row_offset, self.row_offset + b, dtype=torch.float32), te.sum(dim=(1, 2)),
                 images.mean(dim=(1, 2, 3)) if images is not None else torch.zeros(b),
                 mask.reshape(b, -1).float().sum(1) if mask is not None else torch.full((b,), -1.),
                 cond_images.mean(dim=(1, 2, 3)) if cond_images is not None else torch.zeros(b),
                 per_row(kw.get("cond_scale")), per_row(kw.get("temperature")), per_row(kw.get("critic_noise_scale")),
                 torch.full((b,), float(self.sampler_seed % 100003))]
        size = self.image_size
        img = torch.zeros((b, 3 * size * size))
        img[:, :len(feats)] = torch.stack(feats, 1)
        img = img.view(b, 3, size, size)
        if not return_ids:
            return img
        f = self.vae.get_encoded_fmap_size(size)
        return img, torch.arange(self.row_offset, self.row_offset + b)[:, None, None].expand(b, f, f).contiguous()

    def generate(self, texts, cond_images=None, **kw):
        return self._call("generate", texts, cond_images=cond_images, **kw)

    def inpaint(self, texts, images, mask, cond_images=None, **kw):
        return self._call("inpaint", texts, images=images, mask=mask, cond_images=cond_images, **kw)

    def edit(self, texts, images, mask=None, cond_images=None, **kw):
        return self._call("edit", texts, images=images, mask=mask, cond_images=cond_images, **kw)


class StubMuse:
    """Muse.forward itself over two stub stages: the super-resolution stage is conditioned on the base stage's images."""
    forward = Muse.forward

    def __init__(self, base, superres):
        self.base_maskgit, self.superres_maskgit = base, superres


def _inputs(total):
    g = torch.Generator().manual_seed(total)
    te = torch.arange(total * 6, dtype=torch.float32).view(total, 2, 3)
    images = torch.rand((total, 3, 4, 4), generator=g) + torch.arange(total).view(total, 1, 1, 1)
    cond = torch.arange(total, dtype=torch.float32).view(total, 1, 1, 1).expand(total, 3, 2, 2).contiguous()
    pix = torch.rand((total, 4, 4), generator=g) < (torch.arange(total) + 1).view(total, 1, 1) / (total + 1)
    masks = {"pixel_bool": pix, "pixel_4d_01": pix[:, None].float(), "token_bool": pix[:, ::2, ::2].contiguous()}
    settings = dict(cond_scale=[float(i) for i in range(total)], temperature=torch.arange(total, dtype=torch.float32) / 10,
                    critic_noise_scale=0.5)
    return te, images, cond, masks, settings


def _calls(te, images, cond, masks, settings, texts):
    """(name, model maker, call(model, sharded)) of every checked call: sharded=True calls the parallel entry point, False the method."""
    out = []
    out.append(("generate", lambda: StubMaskGit(SEED), lambda m, sh: (parallel.generate_sharded(m, texts, text_embeds=te, cond_images=cond,
               return_ids=True, timesteps=3, **settings) if sh else m.generate(texts, cond_images=cond, return_ids=True, timesteps=3, **settings))))
    for form, mask in masks.items():
        out.append((f"inpaint[{form}]", lambda: StubMaskGit(SEED), (lambda mask: lambda m, sh: (
            parallel.inpaint_sharded(m, texts, images, mask, text_embeds=te, return_ids=True, timesteps=3, **settings) if sh
            else m.inpaint(texts, images, mask, return_ids=True, timesteps=3, **settings)))(mask)))
    out.append(("inpaint[images only]", lambda: StubMaskGit(SEED), lambda m, sh: (
        parallel.inpaint_sharded(m, texts, images, masks["token_bool"], text_embeds=te, cond_scale=2.0) if sh
        else m.inpaint(texts, images, masks["token_bool"], cond_scale=2.0))))
    out.append(("edit[mask=None]", lambda: StubMaskGit(SEED), lambda m, sh: (
        parallel.edit_sharded(m, texts, images, text_embeds=te, return_ids=True, iterations=2, **settings) if sh
        else m.edit(texts, images, return_ids=True, iterations=2, **settings))))
    out.append(("edit[mask]", lambda: StubMaskGit(SEED), lambda m, sh: (
        parallel.edit_sharded(m, texts, images, masks["pixel_4d_01"], text_embeds=te, cond_images=cond, return_ids=True, **settings) if sh
        else m.edit(texts, images, masks["pixel_4d_01"], cond_images=cond, return_ids=True, **settings))))
    return out


def _worker(rank, world, port, total, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    te, images, cond, masks, settings = _inputs(total)
    texts = ["t"] * total
    res = {}
    for name, make, call in _calls(te, images, cond, masks, settings, texts):
        mg = make()
        if rank:
            mg.sampler_seed = None                      # rank 0's seed must reach every rank
        sentinel = mg.transformer.encode_text
        out = call(mg, True)
        assert mg.transformer.encode_text is sentinel and mg.row_offset == 0 and mg.global_batch is None
        assert mg.sampler_seed == (None if rank else SEED)
        res[name] = (tuple(t.numpy() for t in out) if isinstance(out, tuple) else out.numpy(), mg.calls)
    # the cascade: neither stage has a sampler_seed, so rank 0 draws both (base first) and every rank gets them
    torch.manual_seed(100 + rank)
    base, sup = StubMaskGit(), StubMaskGit(image_size=8)
    muse = StubMuse(base, sup)
    hi_res, lo_res = parallel.muse_sharded(muse, texts, text_embeds=te, cond_scale=settings["cond_scale"], temperature=0.7, timesteps=3,
                                           return_lowres=True, return_pil_images=False)
    only = parallel.muse_sharded(muse, texts, text_embeds_shard=te[slice(*parallel.shard_bounds(total, rank, world))], timesteps=3,
                                 return_pil_images=False)
    assert base.sampler_seed is None and sup.sampler_seed is None and base.row_offset == 0 and sup.global_batch is None
    res["muse"] = ((hi_res.numpy(), lo_res.numpy(), only.numpy()), (base.calls, sup.calls))
    q.put((rank, res))                  # by value: a shared tensor's storage would be fetched from this process, which may have exited by then
    dist.barrier()
    dist.destroy_process_group()


def _run(world, total, port):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, total, q)) for r in range(world)]
    for p in procs:
        p.start()
    outs = dict(q.get(timeout=180) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    return outs


def _np(x):
    return tuple(t.numpy() for t in x) if isinstance(x, tuple) else x.numpy()


def _equal(a, b):
    if isinstance(a, tuple):
        return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))
    return a.shape == b.shape and a.dtype == b.dtype and bool((a == b).all())


@pytest.mark.parametrize("world,total,port", [(2, 8, 29641), (2, 7, 29642), (2, 1, 29643), (3, 6, 29644), (3, 7, 29645), (3, 2, 29646)],
                         ids=["w2-even", "w2-uneven", "w2-empty", "w3-even", "w3-uneven", "w3-empty"])
def test_sharded_calls_equal_the_single_process_call(world, total, port):
    outs = _run(world, total, port)
    te, images, cond, masks, settings = _inputs(total)
    texts = ["t"] * total
    for name, make, call in _calls(te, images, cond, masks, settings, texts):
        single = make()
        single.transformer.encode_text = lambda t: te
        want = _np(call(single, False))
        ref_kw = single.calls[0]
        for rank in range(world):
            got, calls = outs[rank][name]
            assert _equal(got, want), (name, rank)
            lo, hi = parallel.shard_bounds(total, rank, world)
            if hi == lo:
                assert calls == [], (name, rank)
                continue
            (seen,) = calls
            assert (seen["seed"], seen["row_offset"], seen["global_batch"]) == (SEED, lo, total), (name, rank)
            for key in ("images", "mask", "cond_images"):           # exactly this rank's rows of every row input
                if ref_kw[key] is None:
                    assert seen[key] is None, (name, key)
                else:
                    assert seen[key].dtype == ref_kw[key].dtype and (seen[key] == ref_kw[key][lo:hi]).all(), (name, rank, key)
            for key, value in ref_kw["settings"].items():
                assert seen["settings"][key] == (value[lo:hi] if isinstance(value, list) else value), (name, rank, key)
    # muse_sharded: equal to Muse.forward in one process under rank 0's torch seed; both stages of every rank use rank 0's two draws of
    # each call, base first
    torch.manual_seed(100)
    seeds = [int(torch.randint(0, 2 ** 62, (1,)).item()) for _ in range(4)]
    base, sup = StubMaskGit(seeds[0]), StubMaskGit(seeds[1], image_size=8)
    base.transformer.encode_text = sup.transformer.encode_text = lambda t: te
    want_hi, want_lo = StubMuse(base, sup).forward(texts, cond_scale=settings["cond_scale"], temperature=0.7, timesteps=3,
                                                   return_lowres=True, return_pil_images=False)
    base.sampler_seed, sup.sampler_seed = seeds[2], seeds[3]
    want_only = StubMuse(base, sup).forward(texts, timesteps=3, return_pil_images=False)
    for rank in range(world):
        (hi_res, lo_res, only), (base_calls, sup_calls) = outs[rank]["muse"]
        assert hi_res.shape == (total, 3, 8, 8) and lo_res.shape == (total, 3, 4, 4), rank
        assert _equal(hi_res, want_hi.numpy()) and _equal(lo_res, want_lo.numpy()) and _equal(only, want_only.numpy()), rank
        lo, hi = parallel.shard_bounds(total, rank, world)
        assert len(base_calls) == len(sup_calls) == (2 if hi > lo else 0)
        for i, (cb, cs) in enumerate(zip(base_calls, sup_calls)):
            assert (cb["seed"], cb["row_offset"], cb["global_batch"]) == (seeds[2 * i], lo, total), (rank, i)
            assert (cs["seed"], cs["row_offset"], cs["global_batch"]) == (seeds[2 * i + 1], lo, total), (rank, i)
            assert cs["cond_images"].shape == (hi - lo, 3, 4, 4)          # this rank's own low-res images, not gathered


def test_attributes_restored_when_the_call_raises():
    mg = StubMaskGit(seed=None, fail=True)
    sentinel = mg.transformer.encode_text
    te, images, _, masks, _ = _inputs(5)
    for call in (lambda: parallel.generate_sharded(mg, ["t"] * 5, text_embeds=te),
                 lambda: parallel.inpaint_sharded(mg, ["t"] * 5, images, masks["token_bool"], text_embeds=te, seed=3),
                 lambda: parallel._run_shard(mg.edit, (mg,), ["t"] * 5, 1, 4, 5, None, text_embeds=te, images=images)):
        with pytest.raises(RuntimeError, match="stub failure"):
            call()
        assert mg.transformer.encode_text is sentinel and mg.row_offset == 0 and mg.global_batch is None and mg.sampler_seed is None
    assert [(c["row_offset"], c["global_batch"]) for c in mg.calls] == [(0, 5), (0, 5), (1, 5)]
    assert mg.calls[1]["seed"] == 3 and mg.calls[2]["images"].shape == (3, 3, 4, 4)
    base, sup = StubMaskGit(seed=1), StubMaskGit(seed=2, image_size=8, fail=True)
    sup.transformer = base.transformer                      # stages sharing one transformer get its encode_text back too
    with pytest.raises(RuntimeError):
        parallel.muse_sharded(StubMuse(base, sup), ["t"] * 2, text_embeds=te[:2])
    assert base.transformer.encode_text is sentinel
    assert (base.sampler_seed, sup.sampler_seed, base.row_offset, sup.row_offset) == (1, 2, 0, 0)


def test_run_shard_by_explicit_bounds_and_empty_shard():
    """The runner takes (lo, hi, total) from its caller (no process group): rows [lo, hi) with row_offset lo, and an empty shard returns
    empty() without calling the model."""
    te, images, _, masks, settings = _inputs(5)
    mg = StubMaskGit(seed=9)
    out, ids = parallel._run_shard(mg.inpaint, (mg,), ["t"] * 5, 2, 5, 5, None, text_embeds=te, images=images, mask=masks["pixel_bool"],
                                   return_ids=True, **settings)
    assert out.shape == (3, 3, 4, 4) and ids[:, 0, 0].tolist() == [2, 3, 4]
    assert (mg.calls[0]["mask"] == masks["pixel_bool"][2:].numpy()).all() and mg.calls[0]["settings"]["cond_scale"] == [2.0, 3.0, 4.0]
    empty = parallel._run_shard(mg.inpaint, (mg,), ["t"] * 5, 5, 5, 5, lambda: parallel._empty_result(mg, True), images=images,
                                mask=masks["pixel_bool"], return_ids=True)
    assert len(mg.calls) == 1
    assert empty[0].shape == (0, 3, 4, 4) and empty[0].dtype == torch.float32
    assert empty[1].shape == (0, 2, 2) and empty[1].dtype == torch.int64


def test_wrong_row_counts_and_aten_edit_raise_before_any_call():
    te, images, _, masks, _ = _inputs(4)
    mg = StubMaskGit(seed=1)
    with pytest.raises(ValueError):
        parallel.inpaint_sharded(mg, ["t"] * 4, images[:3], masks["token_bool"])
    with pytest.raises(ValueError):
        parallel.edit_sharded(mg, ["t"] * 4, images, masks["token_bool"][:2])
    with pytest.raises(ValueError):
        parallel.inpaint_sharded(mg, ["t"] * 4, images, masks["token_bool"], temperature=[1.0] * 3)
    mg.sampler_rng = "aten"
    with pytest.raises(ValueError):
        parallel.edit_sharded(mg, ["t"] * 4, images)
    assert mg.calls == []
