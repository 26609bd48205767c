"""PoseNet's layer chain as two concurrent clip groups (posenet.cu, GroupPlan): the graph forward and the fused sample steps
equal the serial chain that rohm_posenet_profile runs, bit for bit, at every batch split the plan makes; poisoned inputs in
one group's clips never reach the other group's outputs; a second replay repeats the bits; the engine splits the batches
whose QKV GEMM needs more than one wave.  Groups are forced (rohm_posenet_set_option(2, 2)) where the engine's own choice
would keep a small batch serial."""
import contextlib
import ctypes as C
import itertools

import pytest
import torch

from rohm_b200 import synthetic
from rohm_b200.noise_streams import NoiseStreams
from rohm_b200.posenet import PoseNet

pytestmark = pytest.mark.gpu

SHAPES = list(itertools.product((2, 3, 15, 31, 32), (1, 63, 143, 144))) + [(3, 200)]  # T = 200: streaming attention


@pytest.fixture(scope="module")
def posenet(cuda_device):
    m = PoseNet(dataset=synthetic.make_dataset('pose'), body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8,
                num_heads=4, device=cuda_device, traj_feat_dim=22)
    m.load_state_dict({k: v.cpu() for k, v in synthetic.synth_state_dict(m, 1).items()})
    m = m.to(cuda_device).eval()
    m.engine(32, 200, cuda_device)  # one engine serves every shape below
    return m


def _inputs(B, T, seed, dev):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 294, 1, T, generator=g).to(dev)
    cond = synthetic.posenet_batch(B, T, seed)['cond'].to(dev)
    ts = torch.randint(0, 1000, (B,), generator=g).to(dev)
    return x, cond, ts


def _split(B, T):
    """The plan's split point: the fewest 128-row tiles over both groups, ties toward equal halves."""
    S = T + 1
    tiles = lambda k: -(-k * S // 128) + -(-(B - k) * S // 128)
    return min(range(1, B), key=lambda k: (tiles(k), abs(2 * k - B), k))


def _serial(e, x, ts):
    """The forward as rohm_posenet_profile runs it: the serial layer chain on one stream, launched eagerly."""
    B, _, _, T = x.shape
    out = torch.empty_like(x)
    ms, n = (C.c_float * 4)(), (C.c_int * 4)()
    stream = C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
    assert e.lib.rohm_posenet_profile(e.handle, C.c_void_p(x.data_ptr()), C.c_void_p(ts.data_ptr()),
                                      C.c_void_p(out.data_ptr()), B, T, stream, ms, n) == 0
    return out


def _groups(e, mode):
    assert e.lib.rohm_posenet_set_option(e.handle, 2, mode) == 0


@contextlib.contextmanager
def _forced(e, mode):
    _groups(e, mode)
    try:
        yield
    finally:
        _groups(e, 0)


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("B,T", SHAPES)
def test_groups_equal_the_serial_chain(posenet, cuda_device, B, T):
    """Graph forward, fused single-stream step and fused per-clip step as two groups: bit-identical to the serial chain, and
    the steps' x_{t-1} bit-identical to the same steps with the serial chain forced."""
    dev = cuda_device
    x, cond, ts = _inputs(B, T, 1000 * B + T, dev)
    e = posenet.prepare_cond(cond)
    ref = _serial(e, x, ts)
    with _forced(e, 2):
        out = e.forward(x, ts, torch.empty_like(x))
        assert e.launches_per_forward == 86
    assert torch.equal(_bits(out), _bits(ref))
    coef = torch.rand(8, generator=torch.Generator().manual_seed(T)).to(dev)
    gen = torch.cuda.default_generators[dev.index]

    def steps():
        gen.manual_seed(5)
        x0, nxt = e.sample_step(x, ts, coef)
        streams = NoiseStreams([torch.Generator(device=dev).manual_seed(50 + b) for b in range(B)], dev)
        c0, cnxt = e.sample_step(x, ts, coef, streams=streams)
        streams.close()
        return x0, nxt, c0, cnxt

    with _forced(e, 2):
        got = steps()
    with _forced(e, 1):
        want = steps()
    for g, w in zip(got, want):
        assert torch.equal(_bits(g), _bits(w))
    assert torch.equal(_bits(got[0]), _bits(ref)) and torch.equal(_bits(got[2]), _bits(ref))


@pytest.mark.parametrize("B,T,split", [(32, 144, True), (128, 144, True), (32, 143, True), (10, 144, True), (9, 144, False),
                                         (8, 144, False), (2, 144, False), (32, 1, False), (1, 144, False)])
def test_engine_splits_batches_whose_qkv_needs_more_than_one_wave(posenet, cuda_device, B, T, split):
    """The input decides: two groups when the batch's QKV GEMM has more 128 x 128 tiles (12 per row tile) than the 132 SMs
    of an H100 (B = 10 at T = 144: 12 row tiles, 144 tiles), else the serial chain (B = 9: 11 row tiles, 132 tiles).  The
    split forward issues the 8 layers and the output head once per group: 4 + 2 x 41 launches against 4 + 41."""
    if torch.cuda.get_device_properties(cuda_device).multi_processor_count != 132:
        pytest.skip("the tile counts above are those of a 132-SM H100")
    if B > 32:
        posenet.engine(B, T, cuda_device)
    x, cond, ts = _inputs(B, T, 3, cuda_device)
    e = posenet.prepare_cond(cond)
    out = e.forward(x, ts, torch.empty_like(x))
    assert e.launches_per_forward == (86 if split else 45)
    assert torch.equal(_bits(out), _bits(_serial(e, x, ts)))


@pytest.mark.parametrize("B,T", [(32, 144), (31, 143), (3, 200)])
def test_poison_in_one_group_never_reaches_the_other(posenet, cuda_device, B, T):
    """NaN, +-Inf and 1e30 written into every clip of one group's x_t leave every bit of the other group's outputs as they
    were, both ways round.  A tensor map or a stored row that crossed the group boundary would carry them over."""
    x, cond, ts = _inputs(B, T, 7 + B, cuda_device)
    e = posenet.prepare_cond(cond)
    k = _split(B, T)
    vals = torch.tensor([float("nan"), float("inf"), float("-inf"), 1e30], device=cuda_device)
    with _forced(e, 2):
        ref = e.forward(x, ts, torch.empty_like(x))
        for poisoned, kept in ((slice(k, B), slice(0, k)), (slice(0, k), slice(k, B))):
            xp = x.clone()
            n = xp[poisoned].numel()
            xp[poisoned] = vals[torch.arange(n, device=cuda_device) % 4].view(xp[poisoned].shape)
            out = e.forward(xp, ts, torch.empty_like(x))
            assert torch.equal(_bits(out[kept]), _bits(ref[kept]))
            assert not torch.isfinite(out[poisoned][:, 22:]).all()  # the poison did run through its own group
        again = e.forward(x, ts, torch.empty_like(x))
    assert torch.equal(_bits(again), _bits(ref))


def test_second_replay_repeats_the_bits(posenet, cuda_device):
    B, T = 15, 143
    x, cond, ts = _inputs(B, T, 21, cuda_device)
    e = posenet.prepare_cond(cond)
    with _forced(e, 2):
        first = e.forward(x, ts, torch.empty_like(x))
        second = e.forward(x, ts, torch.empty_like(x))
    assert torch.equal(_bits(first), _bits(second))
