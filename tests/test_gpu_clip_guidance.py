"""Guidance with per-clip normalisers (PoseNet.guidance_normaliser = 'clip'): each clip's skating and 2-D projection terms
equal today's kernels on the clip alone, bit for bit, whatever its batch, padding or shard; the guided loops, the sharded
run and the rounds inherit that; the refusals come before any launch; and the default mode keeps its bits."""
import argparse
import ctypes

import pytest
import torch

from oracle import clip_guidance_oracle as cgo
from rohm_b200 import diffusion, parallel, pipeline, synthetic
from rohm_b200._lib import RohmB200Error
from rohm_b200.body_model import kernels_for
from test_gpu_noise_streams import _clone, _gens, _rounds
from test_gpu_posenet_lengths import _bits, _guidance_setup, _model, _poison

pytestmark = pytest.mark.gpu

SK_LENGTHS, SK_T = [143, 60, 2, 1, 143, 97], 143
NO_CONTACT = 1  # a clip with no foot in contact: nothing of it skates


def _no_contact(x, ds, b):
    mean, std = torch.from_numpy(ds.Mean), torch.from_numpy(ds.Std)
    x[b, -4:] = ((0.0 - mean[-4:]) / std[-4:]).reshape(4, 1, 1).to(x.device)
    return x


# ---------------------------------------------------------------------------------------------------------- kernels
def test_skating_per_clip_equals_each_clip_alone(cuda_device):
    dev, B, T = cuda_device, len(SK_LENGTHS), SK_T
    ds, x, m, mean, std, k = _guidance_setup(dev, B, T, 2)
    x = _no_contact(x, ds, NO_CONTACT)
    xg = x.to(dev)
    for lengths in (SK_LENGTHS, None):
        xin = _poison(xg, lengths) if lengths is not None else xg
        L = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device=dev)
        got, loss = k.skating_guidance(xin, mean, std, want_loss=True, lengths=L, per_clip=True)
        assert loss.shape == (B, 4)
        skating = 0
        for b, n in enumerate(lengths or [T] * B):
            alone, aloss = k.skating_guidance(xin[b:b + 1, ..., :n].contiguous(), mean, std, want_loss=True)
            assert torch.equal(_bits(got[b:b + 1, ..., :n]), _bits(alone)), (lengths, b, n)
            assert bool((got[b, ..., n:] == 0).all()), (lengths, b)
            assert float(loss[b, 1]) == float(aloss[1]) and float(loss[b, 3]) == float(aloss[3]), (lengths, b)  # exact counts
            skating += int(float(alone.abs().max()) > 0)
        assert float(got[NO_CONTACT].abs().max()) == 0 and float(loss[NO_CONTACT, 1]) == 0 and float(loss[NO_CONTACT, 3]) == 0
        assert skating >= 3, "too few clips skate for the comparison to mean anything"
        ref = cgo.guide_skating_per_clip(x.double(), torch.from_numpy(ds.Mean).double(), torch.from_numpy(ds.Std).double(),
                                         synthetic.smplx_like_model(0), lengths)
        scale = float(ref.abs().max())
        assert scale > 0 and float((got.cpu().double() - ref).abs().max()) < 2e-4 * scale, lengths
    # the PoseNet hook passes the mode through
    m.guidance_normaliser = 'clip'
    batch = {'lengths': torch.tensor(SK_LENGTHS, device=dev)}
    hook = m.guide_skating_with_smpl(batch, {'pred_xstart': _poison(xg, SK_LENGTHS)}, None, compute_grad='x_0')
    direct = k.skating_guidance(_poison(xg, SK_LENGTHS), mean, std, lengths=torch.tensor(SK_LENGTHS, dtype=torch.int32,
                                                                                          device=dev), per_clip=True)
    assert torch.equal(_bits(hook), _bits(direct))


def _camera(ds, B, kp_frames, seed, dev):
    g = torch.Generator().manual_seed(seed)
    ds.cam_R = torch.tensor([[1., 0, 0], [0, 0, 1], [0, -1, 0]]).to(dev)
    ds.cam_t = torch.tensor([[0.2, -5.0, 1.0]]).to(dev)
    tm = torch.eye(4).repeat(B, 1, 1)
    tm[:, :3, 3] = 0.1 * torch.randn(B, 3, generator=g)
    focal = torch.tensor([[1000., 990.]]).repeat(B, 1) + torch.arange(B)[:, None]
    center = torch.tensor([[900., 500.]]).repeat(B, 1) - torch.arange(B)[:, None]
    kp = torch.cat([900 + 300 * torch.randn(B, kp_frames, 22, 1, generator=g),
                    500 + 200 * torch.randn(B, kp_frames, 22, 1, generator=g),
                    torch.rand(B, kp_frames, 22, 1, generator=g)], dim=-1)
    return {'transf_matrix': tm.to(dev), 'focal_length': focal.to(dev), 'camera_center': center.to(dev),
            'keypoints_2d': kp.to(dev)}


def _nan_past(kp, lengths):
    kp = kp.clone()
    for b, n in enumerate(lengths):
        kp[b, n:] = float("nan")
    return kp


def test_projection_per_clip_equals_each_clip_alone(cuda_device):
    dev, B, T = cuda_device, len(SK_LENGTHS), SK_T
    ds, x, m, mean, std, k = _guidance_setup(dev, B, T, 4)
    cam = _camera(ds, B, T + 5, 9, dev)  # keypoints longer than the clips
    xg = x.to(dev)
    for lengths in (SK_LENGTHS, None):
        m.guidance_normaliser = 'clip'
        batch = dict(cam)
        xin = xg
        if lengths is not None:
            batch['lengths'] = torch.tensor(lengths, device=dev)
            batch['keypoints_2d'] = _nan_past(cam['keypoints_2d'], lengths)
            xin = _poison(xg, lengths)
        got = m.guide_2d_projection_with_smpl(batch, {'pred_xstart': xin}, None, compute_grad='x_0')
        m.guidance_normaliser = 'batch'
        for b, n in enumerate(lengths or [T] * B):
            one = {key: v[b:b + 1] for key, v in batch.items() if key != 'lengths'}
            alone = m.guide_2d_projection_with_smpl(one, {'pred_xstart': xin[b:b + 1, ..., :n].contiguous()}, None,
                                                    compute_grad='x_0')
            assert torch.equal(_bits(got[b:b + 1, ..., :n]), _bits(alone)), (lengths, b, n)
            assert bool((got[b, ..., n:] == 0).all()), (lengths, b)
        assert bool(torch.isfinite(got).all())
        ref, _ = cgo.guide_projection_per_clip(
            x.double(), torch.from_numpy(ds.Mean).double(), torch.from_numpy(ds.Std).double(), synthetic.smplx_like_model(0),
            cam['transf_matrix'].cpu().double(), ds.cam_R.cpu().double(), ds.cam_t.cpu().double(),
            cam['focal_length'].cpu().double(), cam['camera_center'].cpu().double(), cam['keypoints_2d'].cpu().double(),
            lengths)
        scale = float(ref.abs().max())
        assert scale > 0 and float((got.cpu().double() - ref).abs().max()) < 2e-4 * scale, lengths
    # per-clip loss sums through the wrapper: one per clip, each the clip alone's
    aff = m._camera_affine(cam, dev)
    f32 = lambda t: t.float().contiguous()
    L = torch.tensor(SK_LENGTHS, dtype=torch.int32, device=dev)
    _, loss = k.projection_guidance(xg, mean, std, aff, f32(cam['focal_length']), f32(cam['camera_center']),
                                    f32(cam['keypoints_2d']), want_loss=True, lengths=L, per_clip=True)
    assert loss.shape == (B,) and bool((loss > 0).all())


# ---------------------------------------------------------------------------------------------------------- loops
GUIDED_RESPACING = "6" + ",0" * 19  # 6 steps, all at t < 50: every step guided under both schedules
LOOP_LENGTHS, LOOP_T, LOOP_SEEDS = [1, 7, 97, 143], 143, [41, 42, 43, 44]


def _guided_diff(dev):
    a = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    return diffusion.create_gaussian_diffusion(a, diffusion, diffusion.SpacedDiffusionPoseNet, 1000, GUIDED_RESPACING, dev)


@pytest.fixture(scope="module")
def guided_model(cuda_device):
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    return _model(cuda_device, ds)


def _loop_batch(m, dev, grad_type, lengths=LOOP_LENGTHS, T=LOOP_T):
    B = len(lengths)
    batch = {'cond': synthetic.posenet_batch(B, T, 3)['cond'].to(dev), 'lengths': torch.tensor(lengths, device=dev)}
    if grad_type == 'prox':
        cam = _camera(m.dataset, B, T + 2, 11, dev)
        cam['keypoints_2d'] = _nan_past(cam['keypoints_2d'], lengths)
        batch.update(cam)
    return batch


def _one_clip(batch, b, n):
    one = {}
    for key, v in batch.items():
        if key == 'lengths':
            continue
        one[key] = v[b:b + 1, ..., :n].contiguous() if key == 'cond' else v[b:b + 1]
    return one


@pytest.mark.parametrize("grad_type,early_stop", [('amass', False), ('prox', True)])
def test_guided_loop_clip_equals_clip_alone(guided_model, cuda_device, grad_type, early_stop):
    m, dev = guided_model, cuda_device
    B, T = len(LOOP_LENGTHS), LOOP_T
    batch = _loop_batch(m, dev, grad_type)
    gens = _gens(dev, LOOP_SEEDS)
    m.guidance_normaliser = 'clip'
    try:
        out = _guided_diff(dev).p_sample_loop(m, dict(batch, generators=gens), [B, 294, 1, T], clip_denoised=False,
                                              cond_fn_with_grad=True, grad_type=grad_type, early_stop=early_stop)
    finally:
        m.guidance_normaliser = 'batch'
    finite = 0
    for b, n in enumerate(LOOP_LENGTHS):
        one = dict(_one_clip(batch, b, n), generators=_gens(dev, [LOOP_SEEDS[b]]))
        alone = _guided_diff(dev).p_sample_loop(m, one, [1, 294, 1, n], clip_denoised=False, cond_fn_with_grad=True,
                                                grad_type=grad_type, early_stop=early_stop)
        assert torch.equal(_bits(out[b:b + 1, ..., :n]), _bits(alone)), (grad_type, b, n)
        if not early_stop:
            assert bool((out[b, ..., n:] == 0).all()), (grad_type, b)
        finite += int(bool(torch.isfinite(alone).all()))
    print(f"{grad_type}: {finite} of {B} guided clips finite")


def test_sharded_clip_guidance_equals_unsharded_without_a_collective(guided_model, cuda_device):
    m, dev = guided_model, cuda_device
    B, T = len(LOOP_LENGTHS), LOOP_T
    batch = _loop_batch(m, dev, 'amass')
    kw = dict(clip_denoised=False, compute_loss=False, cond_fn_with_grad=True, grad_type='amass')
    m.guidance_normaliser = 'clip'
    try:
        assert getattr(m, "guidance_sum_reducer", None) is None
        full = _guided_diff(dev).eval_losses(m, dict(batch, generators=_gens(dev, LOOP_SEEDS)), [B, 294, 1, T], **kw)[1]
        gens, world, parts = _gens(dev, LOOP_SEEDS), 2, []
        for rank in range(world):
            local = parallel.shard_batch(dict(batch, generators=gens), rank, world, B)
            local['generators'] = parallel.shard_generators(gens, rank, world)
            lo, hi = parallel.shard_bounds(B, rank, world)
            parts.append(_guided_diff(dev).eval_losses(m, local, [hi - lo, 294, 1, T], **kw)[1])
    finally:
        m.guidance_normaliser = 'batch'
    assert torch.equal(_bits(torch.cat(parts)), _bits(full))


# ---------------------------------------------------------------------------------------------------------- rounds
@pytest.fixture(scope="module")
def rounds_nets(cuda_device):
    import test_gpu_pipeline as tp
    from rohm_b200.body_model import BodyModel
    from test_gpu_pipeline_lengths import _datasets
    ds_p, ds_t = _datasets()
    mp, mt, mc, *_ = tp._models(cuda_device, ds_p, ds_t)
    return ds_p, ds_t, mp, mt, mc, BodyModel.create('', device=cuda_device, seed=0)


def test_guided_rounds_clip_equals_recording_alone(rounds_nets, cuda_device):
    dev, lengths, T = cuda_device, [144, 64, 32, 16], 144
    mp = rounds_nets[2]
    gens = _gens(dev, [81, 82, 83, 84])
    clones = [_clone(g) for g in gens]
    mp.guidance_normaliser = 'clip'
    try:
        outs = _rounds(rounds_nets, dev, lengths, T, gens, cond_fn_with_grad=True)
        for b, n in enumerate(lengths):
            one = _rounds(rounds_nets, dev, lengths, T, [clones[b]], clip=b, cond_fn_with_grad=True)
            for i, (x, y) in enumerate(zip(outs, one)):
                assert torch.equal(_bits(x[b:b + 1]), _bits(y)), f"recording {b} ({n} frames), output {i}"
    finally:
        mp.guidance_normaliser = 'batch'
    assert all(bool(torch.isfinite(t).all()) for t in outs)


# ---------------------------------------------------------------------------------------------------------- refusals
def test_refusals_come_before_any_launch(rounds_nets, cuda_device):
    dev = cuda_device
    m = _model(dev)
    batch = {'cond': torch.zeros(2, 294, 1, 16, device=dev), 'lengths': torch.tensor([16, 9], device=dev)}
    m.guidance_normaliser = 'per-clip'
    with pytest.raises(RohmB200Error, match="guidance_normaliser"):
        _guided_diff(dev).p_sample_loop(m, batch, [2, 294, 1, 16], cond_fn_with_grad=True, grad_type='amass')
    m.guidance_normaliser = 'clip'
    with pytest.raises(RohmB200Error, match="guidance_normaliser='clip'"):
        parallel.global_guidance(m)
    m.guidance_sum_reducer = lambda s: s
    with pytest.raises(RohmB200Error, match="global_guidance"):
        _guided_diff(dev).p_sample_loop(m, batch, [2, 294, 1, 16], cond_fn_with_grad=True, grad_type='amass')
    assert m._engine is None
    # run_rounds replays the AMASS driver: 'prox' with lengths stays refused in 'clip' mode
    import test_gpu_pipeline as tp
    ds_p, ds_t, mp, mt, mc, bm = rounds_nets
    dp, dt, dc = tp._diffusions(dev, 4, pose_respacing="3" + ",0" * 19)
    pose, traj = synthetic.pipeline_batches(2, 5, ds_p, frames=144, device=dev)
    traj['lengths'] = torch.tensor([144, 64], device=dev)
    seen = []
    mp.guidance_normaliser = 'clip'
    try:
        with pytest.raises(RohmB200Error, match="prox"):
            pipeline.run_rounds(pipeline.make_args(), mp, mt, mc, dp, dt, dc, ds_p, ds_t, bm, pose, traj, grad_type='prox',
                                on_round=lambda *a: seen.append(a))
    finally:
        mp.guidance_normaliser = 'batch'
    assert not seen and 'lengths' not in pose
    # the C entry point: lengths without per-clip normalisers
    k = kernels_for(bm, dev, 32, with_vertices=False)
    z = torch.zeros(2, 294, 1, 16, device=dev)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    L = torch.tensor([16, 9], dtype=torch.int32, device=dev)
    rc = k.lib.rohm_projection_guidance(k.handle, p(z), p(z), p(z), p(L), 2, 16, 0, p(z), p(z), p(z), p(z), 16, p(z),
                                        ctypes.c_void_p(0), k._stream())
    assert rc != 0 and "per_clip" in k.lib.rohm_last_error(k.ctx).decode()
    with pytest.raises(RohmB200Error, match="per_clip"):
        k.projection_guidance(z, z, z, z, z, z, z, lengths=L)


# ---------------------------------------------------------------------------------------------------------- default
def test_batch_mode_set_explicitly_keeps_the_default_bits(guided_model, cuda_device):
    m, dev = guided_model, cuda_device
    B, T = 3, 64
    batch = _loop_batch(m, dev, 'prox', lengths=[T] * B, T=T)
    del batch['lengths']
    outs = []
    for mode in ('unset', 'batch'):
        if mode == 'unset':
            del m.guidance_normaliser
        else:
            m.guidance_normaliser = mode
        d = _guided_diff(dev)
        outs.append(d.p_sample_loop(m, dict(batch, generators=_gens(dev, LOOP_SEEDS[:B])), [B, 294, 1, T],
                                    clip_denoised=False, cond_fn_with_grad=True, grad_type='prox'))
    m.guidance_normaliser = 'batch'
    assert torch.equal(_bits(outs[0]), _bits(outs[1]))
