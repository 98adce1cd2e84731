"""CPU: parsing of `image_seeds`, its ValueErrors, the uint64 <-> int64 bit mapping, splitmix64, and the shard runner's slicing."""
import types

import pytest
import torch

from muse_maskgit_pytorch_b200 import parallel
from muse_maskgit_pytorch_b200.muse_maskgit import MaskGit, _image_seeds, _seed_bits, splitmix64

U64 = 1 << 64


def test_single_int_expands_to_consecutive_seeds():
    assert _image_seeds(42, 4) == (42, 43, 44, 45)
    assert _image_seeds(U64 - 2, 3) == (U64 - 2, U64 - 1, 0)            # mod 2^64
    assert _image_seeds(None, 3) is None


def test_sequences_and_tensors():
    assert _image_seeds([0, U64 - 1, 5], 3) == (0, U64 - 1, 5)
    assert _image_seeds((7, 8), 2) == (7, 8)
    assert _image_seeds(torch.tensor([3, 4], dtype=torch.int32), 2) == (3, 4)
    assert _image_seeds(torch.tensor([-1, -(1 << 63), 9]), 3) == (U64 - 1, 1 << 63, 9)    # int64: two's-complement bits of a uint64


def test_bit_mapping_round_trips():
    seeds = (0, 1, (1 << 63) - 1, 1 << 63, U64 - 1)
    bits = _seed_bits(seeds)
    assert bits.dtype == torch.int64
    assert bits.tolist() == [0, 1, (1 << 63) - 1, -(1 << 63), -1]
    assert _image_seeds(bits, len(seeds)) == seeds


@pytest.mark.parametrize("value,b", [
    ([1, 2], 3),                                  # wrong length
    (torch.tensor([1, 2, 3]), 2),
    ([1, -1], 2),                                 # outside [0, 2^64)
    ([1, U64], 2),
    (-1, 2),
    (U64, 2),
    (torch.tensor([1, -2], dtype=torch.int32), 2),
    (torch.tensor([1.0, 2.0]), 2),                # non-integer dtypes
    (torch.tensor([True, False]), 2),
    ([1.0, 2.0], 2),
    ([True, False], 2),
    (True, 2),
    (1.5, 2),
    (torch.tensor([[1, 2]]), 2),                  # not 1-D
    ("12", 2),
])
def test_bad_values_raise(value, b):
    with pytest.raises(ValueError):
        _image_seeds(value, b)


def test_splitmix64_hand_computed():
    # state 0: z = 0x9E3779B97F4A7C15; z ^= z >> 30, z *= 0xBF58476D1CE4E5B9; z ^= z >> 27, z *= 0x94D049BB133111EB; z ^= z >> 31
    z = 0x9E3779B97F4A7C15
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) % U64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) % U64
    assert splitmix64(0) == z ^ (z >> 31) == 0xE220A8397B1DCDAF      # the first output of SplitMix64 seeded with 0
    assert splitmix64(U64 - 0x9E3779B97F4A7C15) == 0                  # state + gamma = 0 mod 2^64 mixes to 0
    assert all(0 <= splitmix64(s) < U64 for s in (1, 42, U64 - 1))


def _stub(sampler_rng="mmg", noise_fn=None):
    return types.SimpleNamespace(sampler_rng=sampler_rng, sampler_noise_fn=noise_fn)


def test_call_errors_where_no_per_image_stream_exists():
    with pytest.raises(ValueError, match="aten"):
        MaskGit._image_seeds_arg(_stub("aten"), [1, 2], 2)
    with pytest.raises(ValueError, match="sampler_noise_fn"):
        MaskGit._image_seeds_arg(_stub(noise_fn=lambda step, shape: None), [1, 2], 2)
    assert MaskGit._image_seeds_arg(_stub("aten"), None, 2) is None
    assert MaskGit._image_seeds_arg(_stub(), 10, 2) == (10, 11)


class _Recorder:
    """A stand-in for a MaskGit: records the call and the attributes _run_shard sets."""
    def __init__(self):
        self.transformer = types.SimpleNamespace(encode_text=None)
        self.row_offset, self.global_batch, self.sampler_seed = 0, None, None
        self.calls = []

    def method(self, texts, **kw):
        self.calls.append(dict(texts=list(texts), sampler_seed=self.sampler_seed, **kw))
        return "result"


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("seeds", [[11, 12, 13, 14, 15, 16, 17], 100, torch.tensor([-1, 2, 3, 4, 5, 6, 7])])
def test_run_shard_slices_image_seeds_by_global_row(world, seeds):
    total = 7
    texts = [str(i) for i in range(total)]
    full = _image_seeds(seeds, total)
    got = []
    state = torch.get_rng_state()
    for rank in range(world):
        lo, hi = parallel.shard_bounds(total, rank, world)
        m = _Recorder()
        parallel._run_shard(m.method, (m,), texts, lo, hi, total, lambda: None, image_seeds=seeds)
        call = m.calls[0]
        assert call["texts"] == texts[lo:hi] and call["sampler_seed"] is None and m.sampler_seed is None
        assert tuple(call["image_seeds"]) == full[lo:hi]
        got.extend(call["image_seeds"])
    assert tuple(got) == full
    assert torch.equal(torch.get_rng_state(), state)              # no call seed drawn with per-image seeds


def test_run_shard_checks_image_seeds_on_the_whole_batch():
    m = _Recorder()
    with pytest.raises(ValueError):
        parallel._run_shard(m.method, (m,), ["a"] * 4, 0, 2, 4, lambda: None, image_seeds=[1, 2, 3])
    assert not m.calls
