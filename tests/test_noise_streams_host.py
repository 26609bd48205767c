"""Host-side checks of batch['generators'] (rohm_b200.noise_streams.check_generators) and the sharding helper; no GPU."""
import types

import pytest
import torch

from rohm_b200 import parallel
from rohm_b200._lib import RohmB200Error
from rohm_b200.noise_streams import MAX_CLIPS, check_generators


def test_no_key_is_no_streams():
    assert check_generators({}, 3, "cuda:0") is None
    assert check_generators({'generators': None}, 3, "cuda:0") is None


@pytest.mark.parametrize("gens,match", [
    ("not a list", "list or tuple"),
    ([torch.Generator()], "1 generators for a batch of 2"),
    ([torch.Generator(), 3], "not a torch.Generator"),
    ([torch.Generator(), torch.Generator()], "cpu generator"),
])
def test_bad_generators_are_refused(gens, match):
    with pytest.raises(RohmB200Error, match=match):
        check_generators({'generators': gens}, 2, "cuda:0")


def test_the_same_generator_twice_is_refused():
    g = torch.Generator()
    with pytest.raises(RohmB200Error, match="twice"):
        check_generators({'generators': [g, g]}, 2, "cuda:0")


def test_too_many_clips_are_refused():
    gens = [torch.Generator() for _ in range(MAX_CLIPS + 1)]
    with pytest.raises(RohmB200Error, match=f"at most {MAX_CLIPS}"):
        check_generators({'generators': gens}, MAX_CLIPS + 1, "cuda:0")


def test_const_noise_and_replaced_noise_sources_are_refused():
    gens = [torch.Generator(), torch.Generator()]
    with pytest.raises(RohmB200Error, match="const_noise"):
        check_generators({'generators': gens}, 2, "cuda:0", const_noise=True)
    taped = types.SimpleNamespace(_randn=lambda *a, **k: None, _randn_like=torch.randn_like)
    with pytest.raises(RohmB200Error, match="replaced noise source"):
        check_generators({'generators': gens}, 2, "cuda:0", diffusion=taped)
    sharded = parallel.ShardedNoise(4, 0, 2).install(types.SimpleNamespace())
    with pytest.raises(RohmB200Error, match="replaced noise source"):
        check_generators({'generators': gens}, 2, "cuda:0", diffusion=sharded)


@pytest.mark.parametrize("n,world", [(4, 1), (4, 2), (5, 3), (2, 4)])
def test_shard_generators_follows_shard_bounds(n, world):
    gens = [object() for _ in range(n)]
    got = [parallel.shard_generators(gens, r, world) for r in range(world)]
    assert [x for part in got for x in part] == gens
    for r, part in enumerate(got):
        lo, hi = parallel.shard_bounds(n, r, world)
        assert part == gens[lo:hi] and isinstance(part, list)
    assert parallel.shard_generators(tuple(gens), 0, 1) == gens
