"""Per-clip noise streams (batch['generators']): the draw kernel and the fused update against torch's own per-clip draws,
bit for bit; PoseNet, TrajNet / TrajControl and the rounds giving each clip what it gets alone with its generator, in any
batch; fused and unfused paths agreeing; the sharding helper; and the refusals."""
import argparse

import pytest
import torch

from rohm_b200 import diffusion, ops, parallel, pipeline, synthetic
from rohm_b200._lib import RohmB200Error
from rohm_b200.noise_streams import NoiseStreams

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32)


def _gens(dev, seeds, offsets=None):
    out = []
    for i, s in enumerate(seeds):
        g = torch.Generator(device=dev)
        g.manual_seed(s)
        if offsets is not None:
            g.set_offset(offsets[i])
        out.append(g)
    return out


def _clone(g):
    c = torch.Generator(device=g.device)
    c.set_state(g.get_state())
    return c


def _alone_shape(layout, C, n):
    return (1, C, 1, n) if layout == "pose" else (1, n, C)


def _frames(t, layout, b, lo, hi=None):
    return t[b:b + 1, ..., lo:hi] if layout == "pose" else t[b:b + 1, lo:hi]


class _ClipTape:
    """A noise source that builds every padded draw from torch.randn(S_b, generator=clone_b), zero past each clip."""

    def __init__(self, gens, lengths, layout, dev):
        self.gens, self.lengths, self.layout, self.dev, self.calls = gens, lengths, layout, dev, 0

    def _draw(self, shape):
        self.calls += 1
        out = torch.zeros(tuple(shape), device=self.dev)
        C = shape[1] if self.layout == "pose" else shape[2]
        T = shape[-1] if self.layout == "pose" else shape[1]
        for b, g in enumerate(self.gens):
            n = T if self.lengths is None else self.lengths[b]
            z = torch.randn(_alone_shape(self.layout, C, n), generator=g, device=self.dev)
            if self.layout == "pose":
                out[b:b + 1, ..., :n] = z
            else:
                out[b:b + 1, :n] = z
        return out

    def randn(self, *shape, device=None, **kw):
        shape = shape[0] if len(shape) == 1 and isinstance(shape[0], (list, tuple)) else shape
        return self._draw(shape)

    def randn_like(self, x):
        return self._draw(x.shape)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("layout,C", [("pose", 294), ("traj", 13), ("traj", 22)])
def test_randn_clips_equals_torch_per_clip(cuda_device, layout, C):
    """Clip b of two consecutive draws equals two torch.randn(S_b, generator=clone_b) calls, bit for bit; padded frames are
    +0; the generators end at torch's offsets.  1000 frames x 294 channels exceed torch's 270336 virtual threads (a thread
    uses more than one of its four normals) and 4999 frames take two curand_normal4 rounds."""
    dev = cuda_device
    lengths = [1, 7, 144, 1000, 4999]
    B, T = len(lengths), max(lengths)
    gens = _gens(dev, [101 + b for b in range(B)], offsets=[0, 4, 8, 400, 12])
    clones = [_clone(g) for g in gens]
    shape = [B, C, 1, T] if layout == "pose" else [B, T, C]
    s = NoiseStreams(gens, dev)
    draws = [ops.randn_clips(s, shape, layout == "traj", tuple(lengths)) for _ in range(2)]
    s.close()
    for out in draws:
        for b, n in enumerate(lengths):
            ref = torch.randn(_alone_shape(layout, C, n), generator=clones[b], device=dev)
            assert torch.equal(_bits(_frames(out, layout, b, 0, n)), _bits(ref)), (layout, C, b, n)
            assert bool((_bits(_frames(out, layout, b, n)) == 0).all()), (layout, b, "padded frames")
    for g, c in zip(gens, clones):
        assert g.get_offset() == c.get_offset()


@pytest.mark.parametrize("layout", ["pose", "traj"])
@pytest.mark.parametrize("per_clip_coef", [False, True])
@pytest.mark.parametrize("n_grads", [0, 1, 2])
def test_fused_update_equals_ddpm_step_on_clip_noise(cuda_device, layout, per_clip_coef, n_grads):
    dev = cuda_device
    lengths = [1, 7, 144, 1000] if layout == "pose" else [16, 48, 144, 1008]
    C = 294 if layout == "pose" else 22
    B, T = len(lengths), max(lengths)
    shape = [B, C, 1, T] if layout == "pose" else [B, T, C]
    g = torch.Generator(device=dev).manual_seed(5)
    x0, xt = torch.randn(shape, generator=g, device=dev), torch.randn(shape, generator=g, device=dev)
    grads = tuple(torch.randn(shape, generator=g, device=dev) for _ in range(n_grads))
    coef = torch.rand((B, 8) if per_clip_coef else (8,), generator=g, device=dev)
    gens = _gens(dev, [7 + b for b in range(B)])
    clones = [_clone(x) for x in gens]
    cl = layout == "traj"
    noise = ops.randn_clips(NoiseStreams(clones, dev), shape, cl, tuple(lengths))
    ref = ops.ddpm_step(x0, xt, noise, coef, grads=grads)
    got = ops.ddpm_step_philox_clips(x0, xt, coef, NoiseStreams(gens, dev), cl, tuple(lengths), grads=grads)
    for b, n in enumerate(lengths):
        assert torch.equal(_bits(_frames(got, layout, b, 0, n)), _bits(_frames(ref, layout, b, 0, n))), (b, n)
        assert bool((_bits(_frames(got, layout, b, n)) == 0).all()), (b, "padded frames")


# ------------------------------------------------------------------------------------------------ PoseNet
@pytest.fixture(scope="module")
def posenet(cuda_device):
    from test_gpu_posenet_lengths import _model
    return _model(cuda_device)


def _pose_diff(dev, steps=1000, respacing='20'):
    a = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    return diffusion.create_gaussian_diffusion(a, diffusion, diffusion.SpacedDiffusionPoseNet, steps, respacing, dev)


POSE_LENGTHS, POSE_T = [1, 7, 144, 160], 160
POSE_SEEDS, POSE_OFFSETS = [31, 32, 33, 34], [0, 8, 40, 4]


def _pose_run(m, d, cond, lengths, gens, T, **kw):
    batch = {'cond': cond, 'lengths': torch.tensor(lengths, device=cond.device), 'generators': gens}
    return d.p_sample_loop(m, batch, [len(lengths), 294, 1, T], clip_denoised=False, **kw)


@pytest.mark.parametrize("steps,respacing", [(1000, '20'), (40, '')])
def test_posenet_fused_clip_equals_clip_alone_on_default_generator(posenet, cuda_device, steps, respacing):
    """No tapes, the fused one-graph step: clip b equals [1, 294, 1, n_b] sampled alone on the default generator in the
    same (seed, offset), and its generator ends at that generator's final offset.  Another clip order, another B and
    another padded T give the same per-clip bits."""
    m, dev = posenet, cuda_device
    d = _pose_diff(dev, steps, respacing)
    cond = synthetic.posenet_batch(4, POSE_T, 3)['cond'].to(dev)
    gens = _gens(dev, POSE_SEEDS, POSE_OFFSETS)
    out = _pose_run(m, d, cond, POSE_LENGTHS, gens, POSE_T)
    default = torch.cuda.default_generators[dev.index if dev.index is not None else 0]
    for b, n in enumerate(POSE_LENGTHS):
        default.manual_seed(POSE_SEEDS[b])
        default.set_offset(POSE_OFFSETS[b])
        alone = d.p_sample_loop(m, {'cond': cond[b:b + 1, ..., :n].contiguous()}, [1, 294, 1, n], clip_denoised=False)
        assert torch.equal(_bits(out[b:b + 1, ..., :n]), _bits(alone)), f"clip {b} ({n} frames)"
        assert bool((out[b, ..., n:] == 0).all())
        assert gens[b].get_offset() == default.get_offset(), b
    # the same clips reversed, as a sub-batch, and padded to another T
    for order, T2 in (([3, 2, 1, 0], POSE_T), ([2, 0], POSE_T), ([1, 3, 2], 200)):
        c2 = torch.zeros(len(order), 294, 1, T2, device=dev)
        for i, b in enumerate(order):
            c2[i, ..., :POSE_LENGTHS[b]] = cond[b, ..., :POSE_LENGTHS[b]]
        o2 = _pose_run(m, d, c2, [POSE_LENGTHS[b] for b in order], _gens(dev, [POSE_SEEDS[b] for b in order],
                                                                           [POSE_OFFSETS[b] for b in order]), T2)
        for i, b in enumerate(order):
            n = POSE_LENGTHS[b]
            assert torch.equal(_bits(o2[i:i + 1, ..., :n]), _bits(out[b:b + 1, ..., :n])), (order, T2, b)


def test_posenet_fused_and_unfused_agree(posenet, cuda_device, monkeypatch):
    """ROHM_B200_FUSED_STEP=0 (explicit noise tensor + update) and graphs off give the fused path's bits."""
    m, dev = posenet, cuda_device
    d = _pose_diff(dev)
    cond = synthetic.posenet_batch(4, POSE_T, 3)['cond'].to(dev)
    ref = _pose_run(m, d, cond, POSE_LENGTHS, _gens(dev, POSE_SEEDS, POSE_OFFSETS), POSE_T)
    monkeypatch.setattr(diffusion, "_FUSED_STEP", False)
    unfused = _pose_run(m, d, cond, POSE_LENGTHS, _gens(dev, POSE_SEEDS, POSE_OFFSETS), POSE_T)
    monkeypatch.setattr(diffusion, "_FUSED_STEP", True)
    e = m._engine
    e.lib.rohm_posenet_set_option(e.handle, 0, 0)
    try:
        eager = _pose_run(m, d, cond, POSE_LENGTHS, _gens(dev, POSE_SEEDS, POSE_OFFSETS), POSE_T)
    finally:
        e.lib.rohm_posenet_set_option(e.handle, 0, 1)
    assert torch.equal(_bits(unfused), _bits(ref)) and torch.equal(_bits(eager), _bits(ref))


def test_guided_posenet_loop_equals_clip_tape(posenet, cuda_device):
    """The guided loop (skating guidance on every step, one gradient term in the update) with generators equals the same
    loop driven by a tape of per-clip torch draws, on every real frame; padded frames of the result are zero.  With the
    synthetic weights the 3e6-weighted guidance drives the longer clips to NaN on both paths (the update is ill-conditioned,
    see test_gpu_pipeline.py), so the comparison is of bits, NaN included."""
    m, dev = posenet, cuda_device
    d = _pose_diff(dev)
    cond = synthetic.posenet_batch(4, POSE_T, 3)['cond'].to(dev)
    gens = _gens(dev, POSE_SEEDS, POSE_OFFSETS)
    tape = _ClipTape([_clone(g) for g in gens], POSE_LENGTHS, "pose", dev)
    out = _pose_run(m, d, cond, POSE_LENGTHS, gens, POSE_T, cond_fn_with_grad=True, grad_type='amass')
    dt = _pose_diff(dev)
    dt._randn, dt._randn_like = tape.randn, tape.randn_like
    batch = {'cond': cond, 'lengths': torch.tensor(POSE_LENGTHS, device=dev)}
    ref = dt.p_sample_loop(m, batch, [4, 294, 1, POSE_T], clip_denoised=False, cond_fn_with_grad=True, grad_type='amass')
    assert tape.calls == 21
    for b, n in enumerate(POSE_LENGTHS):
        assert torch.equal(_bits(out[b:b + 1, ..., :n]), _bits(ref[b:b + 1, ..., :n])), b
        assert bool((out[b, ..., n:] == 0).all())
    for g, c in zip(gens, tape.gens):
        assert g.get_offset() == c.get_offset()


# ------------------------------------------------------------------------------------------------ TrajNet / TrajControl
@pytest.fixture(scope="module")
def trajnets(cuda_device):
    from test_gpu_trajnet_lengths import _build
    return {False: _build(False, cuda_device)[0], True: _build(True, cuda_device)[0]}


@pytest.mark.parametrize("control", [False, True])
def test_trajnet_clip_equals_one_clip_batch_and_tape(trajnets, cuda_device, control):
    from test_gpu_trajnet_lengths import _clip, _diff, _inputs
    m, dev = trajnets[control], cuda_device
    lengths, T = [144, 48, 16], 144
    batch, _ = _inputs(len(lengths), T, control, 9, dev)
    del batch['x_t']
    batch['lengths'] = torch.tensor(lengths, device=dev)
    gens = _gens(dev, [61, 62, 63], [0, 12, 4])
    clones = [_clone(g) for g in gens]
    tape = _ClipTape([_clone(g) for g in gens], lengths, "traj", dev)
    out = _diff(dev).p_sample_loop(m, dict(batch, generators=gens), [3, T, 13], clip_denoised=False)
    for b, n in enumerate(lengths):
        one = dict(_clip(batch, b), generators=[clones[b]])
        alone = _diff(dev).p_sample_loop(m, one, [1, T, 13], clip_denoised=False)
        assert torch.equal(_bits(out[b:b + 1]), _bits(alone)), f"clip {b} ({n} frames)"
        assert gens[b].get_offset() == clones[b].get_offset()
    dt = _diff(dev)
    dt._randn, dt._randn_like = tape.randn, tape.randn_like
    ref = dt.p_sample_loop(m, dict(batch), [3, T, 13], clip_denoised=False)
    for b, n in enumerate(lengths):
        assert torch.equal(_bits(out[b:b + 1, :n]), _bits(ref[b:b + 1, :n])), b
        assert bool((out[b, n:] == 0).all())


# ------------------------------------------------------------------------------------------------ rounds
@pytest.fixture(scope="module")
def rounds_nets(cuda_device):
    import test_gpu_pipeline as tp
    from rohm_b200.body_model import BodyModel
    from test_gpu_pipeline_lengths import _datasets
    ds_p, ds_t = _datasets()
    mp, mt, mc, *_ = tp._models(cuda_device, ds_p, ds_t)
    return ds_p, ds_t, mp, mt, mc, BodyModel.create('', device=cuda_device, seed=0)


def _rounds(nets, dev, lengths, T, gens, clip=None, **kw):
    import test_gpu_pipeline as tp
    ds_p, ds_t, mp, mt, mc, bm = nets
    dp, dt, dc = tp._diffusions(dev, 4, pose_steps=1000, pose_respacing="3" + ",0" * 19)
    pose, traj = synthetic.pipeline_batches(len(lengths), 5, ds_p, frames=T, device=dev)
    if clip is not None:
        pose = {k: v[clip:clip + 1].contiguous() for k, v in pose.items()}
        traj = {k: v[clip:clip + 1].contiguous() for k, v in traj.items()}
        lengths = lengths[clip:clip + 1]
    traj['lengths'] = torch.tensor(lengths, device=dev)
    traj['generators'] = gens
    args = pipeline.make_args(sample_iter=2, mask_scheme='lower', **kw)
    outs = pipeline.run_rounds(args, mp, mt, mc, dp, dt, dc, ds_p, ds_t, bm, pose, traj)
    assert pose['generators'] is gens
    return outs


def test_rounds_clip_equals_clip_alone_with_its_generator(rounds_nets, cuda_device):
    dev, lengths, T = cuda_device, [144, 64, 32, 16], 144
    gens = _gens(dev, [71, 72, 73, 74])
    clones = [_clone(g) for g in gens]
    outs = _rounds(rounds_nets, dev, lengths, T, gens, cond_fn_with_grad=False)
    for b, n in enumerate(lengths):
        one = _rounds(rounds_nets, dev, lengths, T, [clones[b]], clip=b, cond_fn_with_grad=False)
        for i, (x, y) in enumerate(zip(outs, one)):
            assert torch.equal(_bits(x[b:b + 1]), _bits(y)), f"clip {b} ({n} frames), output {i}"
        assert gens[b].get_offset() == clones[b].get_offset()
    guided = _rounds(rounds_nets, dev, lengths, T, _gens(dev, [71, 72, 73, 74]), cond_fn_with_grad=True)
    assert all(bool(torch.isfinite(t).all()) for t in guided)


# ------------------------------------------------------------------------------------------------ sharding
def test_sharded_slices_equal_unsharded(posenet, cuda_device):
    """Shards run one after another with their slices of the generators, concatenated, equal the unsharded run."""
    m, dev = posenet, cuda_device
    d = _pose_diff(dev)
    cond = synthetic.posenet_batch(4, POSE_T, 3)['cond'].to(dev)
    L = torch.tensor(POSE_LENGTHS, device=dev)
    full = d.eval_losses(m, {'cond': cond, 'lengths': L, 'generators': _gens(dev, POSE_SEEDS, POSE_OFFSETS)},
                         [4, 294, 1, POSE_T], clip_denoised=False, compute_loss=False)[1]
    gens, world, parts = _gens(dev, POSE_SEEDS, POSE_OFFSETS), 3, []
    batch = {'cond': cond, 'lengths': L, 'generators': gens}
    for rank in range(world):
        local = parallel.shard_batch(batch, rank, world, 4)
        local['generators'] = parallel.shard_generators(gens, rank, world)
        lo, hi = parallel.shard_bounds(4, rank, world)
        parts.append(d.eval_losses(m, local, [hi - lo, 294, 1, POSE_T], clip_denoised=False, compute_loss=False)[1])
    assert torch.equal(_bits(torch.cat(parts)), _bits(full))


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_come_before_any_launch(cuda_device):
    from test_gpu_posenet_lengths import _model
    dev = cuda_device
    m = _model(dev)
    d = _pose_diff(dev)
    cond = synthetic.posenet_batch(2, 16, 3)['cond'].to(dev)
    shape = [2, 294, 1, 16]
    g1, g2 = _gens(dev, [1, 2])
    cases = [([g1], {}, "2 clips"), ([g1, "x"], {}, "not a torch.Generator"), ([g1, g1], {}, "twice"),
             ([g1, torch.Generator()], {}, "cpu generator"), ([g1, g2], {'const_noise': True}, "const_noise")]
    for gens, kw, match in cases:
        with pytest.raises(RohmB200Error, match=match):
            d.p_sample_loop(m, {'cond': cond, 'generators': gens}, shape, clip_denoised=False, **kw)
        assert m._engine is None, match
    tape = _ClipTape([g1, g2], None, "pose", dev)
    d._randn, d._randn_like = tape.randn, tape.randn_like
    with pytest.raises(RohmB200Error, match="replaced noise source"):
        d.p_sample_loop(m, {'cond': cond, 'generators': [g1, g2]}, shape, clip_denoised=False)
    x = torch.zeros(shape, device=dev)
    with pytest.raises(RohmB200Error, match="replaced noise source"):
        d.p_sample(m, {'cond': cond, 'generators': [g1, g2]}, x, torch.zeros(2, dtype=torch.long, device=dev))
    assert tape.calls == 0 and m._engine is None
    assert g1.get_offset() == 0 and g2.get_offset() == 0
