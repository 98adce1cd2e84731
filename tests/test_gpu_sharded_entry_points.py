"""GPU: the sharded entry points give the unsharded call's tokens.  Each test runs parallel._run_shard once per virtual rank of a world
of 2 or 3 (rows [lo, hi) of shard_bounds, the same torch.manual_seed before every call, as every rank of a real group starts from it),
concatenates the shards and compares them with one unsharded call of the same method under the same seed.

Findings asserted here:
  * token ids are identical, in "mmg" mode (one seed for every rank) and "aten" mode (`global_batch`), with and without a token critic,
    also where a shard's largest regenerated-token count N_b, and so its sampled rows per step, differ from the whole batch's;
  * images are bitwise equal to the unsharded call's, which decodes the same ids in one batch: the VAE decode of an image does not
    depend on how many other images share its launch;
  * where the fused tail's column split S of a shard differs from the whole batch's (test_split_count_differs), the ids and images are
    still identical.  S splits the vocabulary columns, so the logits, the candidate lists and the sampled token do not depend on it;
    the confidence score 1 - p divides by a sum of exponentials merged over 2 S segments, whose last bits can depend on S, and a
    score that moved by an ulp could reorder two tokens at the re-mask cut.  No such reordering occurs at these sizes; the test would
    report it as a count of differing ids.
The 2-GPU case runs the public entry points over NCCL when the machine has two devices and is skipped otherwise."""
import os

import pytest
import torch

from muse_maskgit_pytorch_b200 import parallel
from tests import util
from tests.test_gpu_inpaint import _images, _ragged_tokens
from tests.test_gpu_models import M, make_branch_maskgit, make_maskgit

pytestmark = pytest.mark.gpu
torch.set_grad_enabled(False)

SCALES = [3.0, 1.0, 2.0, 5.0, 3.0, 4.0, 1.5]
FRACS = [1, 0.3, 0.6, 0, 0.5, 0.8, 0.2]          # N_b of 16 tokens differ; no shard of 2 or 3 ranks but the first holds the full mask


def _te(b):
    return util.text_embeds("g4.te", 3, 8, 128, 14).cuda().repeat(-(-b // 3), 1, 1)[:b].contiguous()


def _virtual_ranks(method, maskgits, texts, world, seed, **kw):
    """The results of `world` ranks' _run_shard calls, concatenated by row."""
    total = len(texts)
    parts = []
    for rank in range(world):
        lo, hi = parallel.shard_bounds(total, rank, world)
        torch.manual_seed(seed)
        parts.append(parallel._run_shard(method, maskgits, texts, lo, hi, total, None, **kw))
    return tuple(torch.cat(p) for p in zip(*parts))


def _unsharded(method, maskgits, texts, te, seed, **kw):
    for m in maskgits:
        m.transformer.encode_text = lambda t: te
    torch.manual_seed(seed)
    return method(texts, **kw)


def _compare(name, full_ids, shard_ids, full_images, shard_images):
    n_diff = 0 if full_ids is None else int((full_ids != shard_ids).sum())
    same = [torch.equal(a, b) for a, b in zip(full_images, shard_images)]
    err = max(float((a - b).abs().max()) for a, b in zip(full_images, shard_images))
    print(f"{name}: {n_diff} of {0 if full_ids is None else full_ids.numel()} ids differ; images bitwise equal: {same} (max |diff| {err:.3e})")
    assert n_diff == 0, name
    assert all(same), name


@pytest.mark.parametrize("critic", [False, True], ids=["no_critic", "token_critic"])
@pytest.mark.parametrize("rng", ["mmg", "aten"])
@pytest.mark.parametrize("world", [2, 3])
def test_inpaint_virtual_ranks_equal_the_unsharded_call(world, rng, critic):
    if critic:
        mg, kw, _ = make_branch_maskgit("gen_critic_small", "bf16")
        kw = dict(critic_noise_scale=[0.7, 0.2, 1.0, 0.5, 0.0, 0.9, 0.3])
    else:
        mg, kw = make_maskgit("bf16"), {}
    mg.sampler_rng = rng
    b = len(SCALES)
    texts, te, img = ["a"] * b, _te(b), _images(b, 16)
    mask = _ragged_tokens(b, 4, 8, FRACS).cuda()
    counts = mask.reshape(b, -1).sum(1).tolist()
    lo, hi = parallel.shard_bounds(b, 1, world)
    assert max(counts[lo:hi]) < max(counts)                 # rank 1 samples fewer rows per step than the whole batch
    kw.update(cond_scale=SCALES, timesteps=8, return_ids=True)
    full_img, full_ids = _unsharded(mg.inpaint, (mg,), texts, te, 21, images=img, mask=mask, **kw)
    img_s, ids_s = _virtual_ranks(mg.inpaint, (mg,), texts, world, 21, text_embeds=te, images=img, mask=mask, **kw)
    _compare(f"inpaint world {world} {rng} critic={critic}", full_ids, ids_s, [full_img], [img_s])
    assert torch.equal(full_ids.reshape(b, -1)[~mask.reshape(b, -1)], mg.vae.encode_ids(img).reshape(b, -1)[~mask.reshape(b, -1)])


@pytest.mark.parametrize("world", [2, 3])
def test_edit_virtual_ranks_equal_the_unsharded_call(world):
    mg = make_maskgit("bf16")
    b = len(SCALES)
    texts, te, img = ["a"] * b, _te(b), _images(b, 16)
    mask = _ragged_tokens(b, 4, 9, FRACS).cuda()
    kw = dict(mask=mask, iterations=2, fraction=0.5, timesteps=3, cond_scale=SCALES, temperature=torch.linspace(0.5, 1.5, b), return_ids=True)
    full_img, full_ids = _unsharded(mg.edit, (mg,), texts, te, 22, images=img, **kw)
    img_s, ids_s = _virtual_ranks(mg.edit, (mg,), texts, world, 22, text_embeds=te, images=img, **kw)
    _compare(f"edit world {world}", full_ids, ids_s, [full_img], [img_s])


@pytest.mark.parametrize("world", [2, 3])
def test_muse_cascade_virtual_ranks_equal_the_unsharded_call(world):
    """Both stages draw their seeds from torch's generator (base first) and see the shard's text embeddings; the super-resolution stage
    of each virtual rank is conditioned on that rank's own low-res images."""
    base, sup = make_maskgit("bf16"), make_maskgit("bf16", superres=True)
    muse = M().Muse(base=base, superres=sup)
    b = 5
    texts, te = ["a"] * b, _te(b)
    kw = dict(cond_scale=SCALES[:b], timesteps=6, return_lowres=True, return_pil_images=False)
    full_hi, full_lo = _unsharded(muse.forward, (base, sup), texts, te, 23, **kw)
    hi_s, lo_s = _virtual_ranks(muse.forward, (base, sup), texts, world, 23, text_embeds=te, **kw)
    assert hi_s.shape == (b, 3, 32, 32) and lo_s.shape == (b, 3, 16, 16)
    _compare(f"muse world {world}", None, None, [full_hi, full_lo], [hi_s, lo_s])
    assert base.sampler_seed is None and sup.sampler_seed is None and base.row_offset == sup.row_offset == 0


def test_split_count_differs_between_shard_and_batch():
    """300 images of 16 tokens: step 0 samples 4800 rows in the whole batch and 2400 in each of two shards, which the fused tail splits
    over a different number of column ranges S (asserted from the planner).  generate and inpaint (ragged masks, image 0 full, so the
    batch and both shards sample 16 rows per image at step 0) give identical ids and bitwise equal images."""
    from oracle import fused_tail as FT
    units = torch.cuda.get_device_properties(0).multi_processor_count
    b, world = 300, 2
    s_full, s_shard = FT.lf_plan(b * 16, 1024, units)["S"], FT.lf_plan(b // world * 16, 1024, units)["S"]
    print(f"fused-tail split count at step 0: whole batch S = {s_full}, shard S = {s_shard} ({units} SMs)")
    assert s_full != s_shard
    mg = make_maskgit("bf16")
    texts, te, img = ["a"] * b, _te(b), _images(b, 16)
    mask = torch.rand((b, 4, 4), generator=torch.Generator().manual_seed(10)) < 0.6
    mask[0] = mask[b // world] = True
    mask = mask.cuda()
    for name, method, kw in (("generate", mg.generate, dict(timesteps=8, return_ids=True)),
                             ("inpaint", mg.inpaint, dict(images=img, mask=mask, timesteps=8, return_ids=True))):
        full_img, full_ids = _unsharded(method, (mg,), texts, te, 24, **kw)
        img_s, ids_s = _virtual_ranks(method, (mg,), texts, world, 24, text_embeds=te, **kw)
        _compare(f"{name} S {s_full} vs {s_shard}", full_ids, ids_s, [full_img], [img_s])


def _nccl_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    torch.distributed.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    mg = make_maskgit("bf16")
    b = len(SCALES)
    texts, te, img = ["a"] * b, _te(b), _images(b, 16)
    mask = _ragged_tokens(b, 4, 8, FRACS).cuda()
    torch.manual_seed(30 + rank)                # only rank 0's draw may decide the seed
    out = {"inpaint": parallel.inpaint_sharded(mg, texts, img, mask, text_embeds=te, cond_scale=SCALES, timesteps=8, return_ids=True),
           "generate": parallel.generate_sharded(mg, texts, text_embeds=te, timesteps=8, return_ids=True)}
    if rank == 0:
        torch.manual_seed(30)
        mg.transformer.encode_text = lambda t: te
        want = {"inpaint": mg.inpaint(texts, img, mask, cond_scale=SCALES, timesteps=8, return_ids=True),
                "generate": mg.generate(texts, timesteps=8, return_ids=True)}
        q.put({k: all(torch.equal(a, w) for a, w in zip(out[k], want[k])) for k in out})
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two CUDA devices")
def test_two_gpus_nccl_equal_one_gpu():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_nccl_worker, args=(r, 2, 29661, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = q.get(timeout=600)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert got == {"inpaint": True, "generate": True}, got
