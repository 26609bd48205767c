"""The TrajNet -> PoseNet rounds and the reconstruction on batches of recordings with different lengths
(test_batch_traj['lengths']): every glue kernel's lengths instance against the existing entry point on the clip cut to its
own length (bit for bit) and against the glue oracle, the NaN repair inside a clip, the compacted body path, run_rounds
clip by clip against the clip alone, the skating-guided rounds with poisoned padding, the flag variants with
reconstruct_outputs / result_dict, and the refusals."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch

from helpers import ROOT, TOL
from oracle import glue_oracle as go
from oracle import kinematics_oracle as ko
from rohm_b200 import _lib, glue, pipeline, synthetic
from rohm_b200._lib import RohmB200Error
from rohm_b200.body_model import BodyKernels, BodyModel, kernels_for
from rohm_b200.motion_representation import recover_from_repr_smpl, split_repr

gpu = pytest.mark.gpu

NEW_SYMBOLS = ("rohm_traj_glue_lengths", "rohm_traj_repr_from_joints_lengths", "rohm_pose_to_control_cond_lengths",
               "rohm_build_pose_cond_lengths", "rohm_body_from_repr_lengths", "rohm_joints_from_traj_lengths")
SEL13 = [0, 2, 3, 6] + list(range(7, 13)) + list(range(16, 19))
SMALL, LONG = (144, 16, 80, 48), (2064, 1040, 16)  # LONG: clusters of 3 CTAs; a clip ending inside CTA 1; one inside CTA 0


def test_c_abi_exports_the_lengths_entry_points():
    """include/rohm_b200.h <-> the ctypes signature table <-> librohm_b200.so for the entry points of this file."""
    header = open(os.path.join(ROOT, "include", "rohm_b200.h")).read()
    declared = set(re.findall(r"ROHM_API\s+[\w\s\*]+?\b(rohm_\w+)\s*\(", header))
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert name in declared and name in _lib.SIGNATURES and hasattr(lib, name), name


def _bits(t):
    return t.contiguous().view(torch.int32)


def _poison(t, lengths, dim=1):
    """A copy with every frame past a clip filled with NaN, +Inf, -Inf and 1e30 in turn (`dim`: the frame axis)."""
    t = t.clone()
    vals = torch.tensor([float("nan"), float("inf"), float("-inf"), 1e30], device=t.device)
    T = t.shape[dim]
    for b, n in enumerate(lengths):
        if n < T:
            fill = vals[torch.arange(n, T, device=t.device) % 4]
            view = t[b].movedim(dim - 1, -1)
            view[..., n:] = fill
    return t


def _datasets():
    return (synthetic.make_dataset('pose', seed=3, realistic_std=True), synthetic.make_dataset('traj', seed=3, realistic_std=True))


@pytest.fixture(scope="module")
def body(cuda_device):
    return BodyModel.create('', device=cuda_device, seed=0), synthetic.smplx_like_model(0)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the glue kernels one by one
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("lengths", [SMALL, LONG])
def test_traj_to_full_repr_ragged_equals_each_clip_alone(body, cuda_device, lengths):
    bm, model = body
    dev = cuda_device
    ds_p, ds_t = _datasets()
    B, T = len(lengths), max(lengths)
    clean = synthetic.plausible_motion(B, T, 7, ds_t)[:, :, 0].permute(0, 2, 1).contiguous()
    traj = clean[..., SEL13] + 0.05 * torch.randn(B, T, 13, generator=torch.Generator().manual_seed(1))
    L = glue.device_lengths(lengths, dev)
    comp, full = glue.traj_to_full_repr(bm, _poison(traj.to(dev), lengths), _poison(clean.to(dev), lengths), ds_t, ds_p,
                                        lengths=L)
    assert comp.shape == (B, T, 294) and full.shape == (B, T - 1, 22)
    for b, n in enumerate(lengths):
        c1, f1 = glue.traj_to_full_repr(bm, traj[b:b + 1, :n].contiguous().to(dev), clean[b:b + 1, :n].contiguous().to(dev),
                                        ds_t, ds_p)
        assert torch.equal(_bits(comp[b, :n]), _bits(c1[0])) and torch.equal(_bits(full[b, :n - 1]), _bits(f1[0])), (b, n)
        assert bool((comp[b, n:] == 0).all()) and bool((full[b, n - 1:] == 0).all()), (b, n)
        if T <= 144:
            _, f_o = go.traj_to_full_repr(traj[b:b + 1, :n], clean[b:b + 1, :n], ds_t.Mean, ds_t.Std, ds_p.Mean, ds_p.Std, model)
            assert float((full[b, :n - 1].cpu() - f_o[0]).abs().max()) < TOL, (b, n)


@gpu
def test_control_cond_and_pose_cond_ragged(cuda_device):
    dev = cuda_device
    lengths = [n - 1 for n in SMALL]  # pose frames
    B, Tp = len(lengths), max(lengths)
    g = torch.Generator().manual_seed(5)
    pose_out, src, tf = (torch.randn(B, 294, 1, Tp, generator=g), torch.randn(B, Tp, 294, generator=g),
                         torch.randn(B, Tp, 22, generator=g))
    L = glue.device_lengths(lengths, dev)
    cc = glue.pose_to_control_cond(_poison(pose_out.to(dev), lengths, dim=3), Tp + 1, 272, lengths=L)
    lo, hi = torch.tensor([100, 3, 40, 0]), torch.tensor([130, 15, 70, 30])
    keep = glue.channel_keep_mask('upper')
    conds = [glue.build_pose_cond(_poison(src.to(dev), lengths), _poison(tf.to(dev), lengths), keep, zero_contact=True, lengths=L),
             glue.build_pose_cond(_poison(src.to(dev), lengths), _poison(tf.to(dev), lengths), None, lo, hi, True, lengths=L),
             glue.build_pose_cond(_poison(pose_out.to(dev), lengths, dim=3), None, keep, zero_contact=True, lengths=L)]
    for b, n in enumerate(lengths):
        one = pose_out[b:b + 1, ..., :n].contiguous()
        alone = glue.pose_to_control_cond(one.to(dev), n + 1, 272)
        assert torch.equal(_bits(cc[b, :n + 1]), _bits(alone[0])) and bool((cc[b, n + 1:] == 0).all()), (b, n)
        assert torch.equal(alone[0].cpu(), go.pose_to_control_cond(one, n + 1, 272)[0])
        s1, t1 = src[b:b + 1, :n].contiguous(), tf[b:b + 1, :n].contiguous()
        want = [go.build_pose_cond(s1, t1, 'upper', True),
                go.build_pose_cond(s1, t1, 'full', True, lo[b:b + 1], torch.minimum(hi[b:b + 1], torch.tensor([n]))),
                go.build_pose_cond(one[:, :, 0].permute(0, 2, 1), None, 'upper', True)]
        for got, w in zip(conds, want):
            assert torch.equal(got[b, ..., :n].cpu(), w[0]) and bool((got[b, ..., n:] == 0).all()), (b, n)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the NaN repair stays inside the clip
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("where", ["first", "middle", "nowhere"])
def test_nan_repair_stays_inside_the_clip(cuda_device, where):
    """Hips and shoulders collapsed onto one point give a 0/0 forward direction.  In frame 0 of a short clip the repair
    takes frame len-1 (not T-1), in a middle frame its predecessor; the packed inputs hold no frame past a clip, so nothing
    there can be searched or used as a source."""
    dev = cuda_device
    lengths, T = (64, 32, 48), 64
    g = torch.Generator().manual_seed(3)
    clips = [(torch.randn(n, 22, 3, generator=g), 0.3 * torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g))
             for n in lengths]
    bad = {"first": 0, "middle": 11}.get(where)
    if bad is not None:
        clips[1][0][bad, [1, 2, 16, 17]] = clips[1][0][bad, 0].clone()
    m0, s1 = torch.zeros(294, device=dev), torch.ones(294, device=dev)
    L = glue.device_lengths(lengths, dev)
    packed = [torch.cat([c[k] for c in clips]).to(dev) for k in range(3)]
    out = glue.traj_repr_from_joints(*packed, m0, s1, lengths=L, frames=T)
    assert out.shape == (3, T - 1, 22)
    for b, n in enumerate(lengths):
        alone = glue.traj_repr_from_joints(*[c[None].to(dev) for c in clips[b]], m0, s1)
        assert torch.equal(_bits(out[b, :n - 1]), _bits(alone[0])), (where, b)
        assert bool(torch.isfinite(out[b]).all()) and bool((out[b, n - 1:] == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# 3. the compacted body path
# ---------------------------------------------------------------------------------------------------------------------
def _check_compacted_body(dev):
    bm, model = BodyModel.create('', device=dev, seed=0), synthetic.smplx_like_model(0)
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    lengths, T = (9, 2, 5), 9
    x = synthetic.plausible_motion(3, T, 17, ds)
    xl = x[:, :, 0].permute(0, 2, 1).contiguous()
    mean, std = glue.stats_on(ds, dev)
    k = kernels_for(bm, dev, 3 * T, with_vertices=True)
    L = glue.device_lengths(lengths, dev)
    jp, vp = k.from_repr(x.to(dev), mean, std, want_vertices=True)
    full = xl * torch.from_numpy(ds.Std) + torch.from_numpy(ds.Mean)
    jo, vo = ko.joints_from_smplx(ko.split_repr(full), model, return_verts=True)
    for cl, xin in ((False, _poison(x.to(dev), lengths, dim=3)), (True, _poison(xl.to(dev), lengths))):
        j, v = k.from_repr(xin, mean, std, want_vertices=True, channels_last=cl, lengths=L)
        assert j.shape == (sum(lengths), 22, 3) and v.shape == (sum(lengths), 10475, 3)
        for b, (jb, vb) in enumerate(zip(glue.split_clips(j, L), glue.split_clips(v, L))):
            n = lengths[b]
            assert torch.equal(_bits(jb), _bits(jp[b, :n])) and torch.equal(_bits(vb), _bits(vp[b, :n])), (cl, b)
            assert float((jb.cpu() - jo[b, :n]).abs().max()) < 2e-5 and float((vb.cpu() - vo[b, :n]).abs().max()) < TOL
    # capacity counts the clips' frames: a handle for 16 frames takes these 16 although B * T = 27
    small = BodyKernels(bm, dev, sum(lengths), with_vertices=True)
    j2, v2 = small.from_repr(x.to(dev), mean, std, want_vertices=True, lengths=L)
    assert torch.equal(_bits(v2), _bits(v)) and torch.equal(_bits(j2), _bits(j))
    with pytest.raises(RohmB200Error):
        small.from_repr(x.to(dev), mean, std, want_vertices=True)
    # the joint-based recovery modes, packed
    rep = {kk: vv.to(dev) for kk, vv in split_repr(_poison(full.to(dev), lengths)).items()}
    clean = {kk: vv.to(dev) for kk, vv in split_repr(full).items()}
    for mode in ('joint_abs_traj', 'joint_rel_traj'):
        got = glue.split_clips(recover_from_repr_smpl(rep, mode, bm, lengths=L), L)
        for b, n in enumerate(lengths):
            alone = recover_from_repr_smpl({kk: vv[b:b + 1, :n] for kk, vv in clean.items()}, mode, bm)
            assert torch.equal(_bits(got[b]), _bits(alone[0])), (mode, b)
    return True


@gpu
def test_compacted_body_path(cuda_device):
    assert _check_compacted_body(cuda_device)


@gpu
def test_compacted_body_path_two_kernel_lbs():
    code = ("import sys, torch\nsys.path.insert(0, %r); sys.path.insert(0, %r)\nimport test_gpu_pipeline_lengths as t\n"
            "assert t._check_compacted_body(torch.device('cuda:0'))\nprint('ok')\n" % (ROOT, os.path.join(ROOT, "tests")))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, ROHM_B200_FUSED_LBS="0"), capture_output=True,
                       text=True)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


# ---------------------------------------------------------------------------------------------------------------------
# 4.-7. run_rounds / reconstruct_outputs
# ---------------------------------------------------------------------------------------------------------------------
class _BatchTape:
    """Seeded noise for the padded batch, draw by draw; with clip=b every draw is row b of the same padded draw, as the clip
    run as a one-clip batch on its slice of the batch's noise sees it."""

    def __init__(self, seed, B, device, clip=None):
        self.seed, self.B, self.device, self.clip, self.k = seed, B, device, clip, 0

    def _draw(self, shape):
        z = torch.randn((self.B,) + tuple(shape[1:]), generator=torch.Generator().manual_seed(1000 * self.seed + self.k))
        self.k += 1
        if self.clip is not None:
            z = z[self.clip:self.clip + 1]
        return z.contiguous().to(self.device)

    def randn(self, *shape, device=None, **kw):
        return self._draw(shape)

    def randn_like(self, x):
        return self._draw(x.shape)


@pytest.fixture(scope="module")
def nets(cuda_device):
    import test_gpu_pipeline as tp
    ds_p, ds_t = _datasets()
    mp, mt, mc, *_ = tp._models(cuda_device, ds_p, ds_t)
    return ds_p, ds_t, mp, mt, mc, BodyModel.create('', device=cuda_device, seed=0)


def _run(nets, dev, lengths, T, seed=5, poison=True, clip=None, pose_respacing="3" + ",0" * 19, with_key=True, **kw):
    """run_rounds on the ragged batch (or on clip `clip` of it as a one-clip batch with lengths=[L]); returns the outputs,
    the per-round stages and the two batch dicts."""
    import test_gpu_pipeline as tp
    ds_p, ds_t, mp, mt, mc, bm = nets
    B = len(lengths)
    dp, dt, dc = tp._diffusions(dev, 4, pose_steps=1000, pose_respacing=pose_respacing)
    tape_p, tape_t = _BatchTape(seed, B, dev, clip), _BatchTape(seed + 1, B, dev, clip)
    dp._randn, dp._randn_like = tape_p.randn, tape_p.randn_like
    for d in (dt, dc):
        d._randn, d._randn_like = tape_t.randn, tape_t.randn_like
    pose, traj = synthetic.pipeline_batches(B, seed, ds_p, frames=T, device=dev)
    if poison:
        pose = {k: _poison(v, [n - 1 for n in lengths]) for k, v in pose.items()}
        traj = {k: _poison(v, lengths) for k, v in traj.items()}
    if clip is not None:
        pose = {k: v[clip:clip + 1].contiguous() for k, v in pose.items()}
        traj = {k: v[clip:clip + 1].contiguous() for k, v in traj.items()}
        lengths = lengths[clip:clip + 1]
    if with_key:
        traj['lengths'] = torch.tensor(lengths, device=dev)
    torch.manual_seed(seed)  # the 'full' scheme's CPU draw
    args = pipeline.make_args(sample_iter=2, **kw)
    seen = []
    on_round = lambda it, *stages: seen.append([s.detach().clone() for s in stages]) or None
    outs = pipeline.run_rounds(args, mp, mt, mc, dp, dt, dc, ds_p, ds_t, bm, pose, traj, on_round=on_round)
    return args, outs, seen, pose, traj


def _frames_of(t, T):
    """(frame axis, frames of a clip of n trajectory frames) for a tensor of the rounds: trajectory tensors have T frames,
    pose tensors T - 1."""
    ax = 1 if t.dim() == 3 else 3
    return ax, (0 if t.shape[ax] == T else 1)


def _assert_zero_past(t, lengths, T):
    ax, less = _frames_of(t, T)
    for b, n in enumerate(lengths):
        assert bool((t[b].movedim(ax - 1, 0)[n - less:] == 0).all()), (tuple(t.shape), b)


@gpu
def test_rounds_without_guidance_equal_each_clip_alone(nets, cuda_device):
    dev, lengths, T = cuda_device, list(SMALL), 144
    _, outs, seen, pose, traj = _run(nets, dev, lengths, T, cond_fn_with_grad=False)
    assert outs[0].shape == (4, 294, 1, 143) and outs[1].shape == (4, 144, 13) and outs[2].shape == (4, 144, 22)
    assert torch.equal(pose['lengths'].cpu(), torch.tensor(lengths) - 1)
    assert pose['cond'].shape == (4, 294, 1, 143) and traj['control_cond'].shape == (4, 144, 272)
    everything = list(outs) + [s for r in seen for s in r] + [pose['cond'], traj['control_cond'], traj['motion_repr_noisy']]
    for t in everything:
        _assert_zero_past(t, lengths, T)
    for b, n in enumerate(lengths):
        _, o1, s1, p1, t1 = _run(nets, dev, lengths, T, clip=b, cond_fn_with_grad=False)
        ragged = list(outs) + [s for r in seen for s in r] + [pose['cond'], traj['control_cond'], traj['motion_repr_noisy']]
        alone = list(o1) + [s for r in s1 for s in r] + [p1['cond'], t1['control_cond'], t1['motion_repr_noisy']]
        for i, (x, y) in enumerate(zip(ragged, alone)):
            assert torch.equal(_bits(x[b:b + 1]), _bits(y)), f"clip {b} ({n} frames), tensor {i}"


@gpu
def test_guided_rounds_ignore_padding_and_uniform_lengths_equal_no_key(nets, cuda_device):
    dev, lengths, T = cuda_device, list(SMALL), 144
    resp = "12" + ",0" * 19  # reaches the guided steps (t <= 50)
    _, a, seen_a, *_ = _run(nets, dev, lengths, T, poison=False, pose_respacing=resp)
    _, b, seen_b, *_ = _run(nets, dev, lengths, T, poison=True, pose_respacing=resp)
    for x, y in zip(list(a) + [s for r in seen_a for s in r], list(b) + [s for r in seen_b for s in r]):
        assert torch.equal(_bits(x), _bits(y)), "values in padded frames reached an output"
        assert bool(torch.isfinite(x).all())
        _assert_zero_past(x, lengths, T)
    _, u, *_ = _run(nets, dev, [T] * 2, T, poison=False, pose_respacing=resp)
    _, v, *_ = _run(nets, dev, [T] * 2, T, poison=False, pose_respacing=resp, with_key=False)
    for x, y in zip(u, v):
        assert torch.equal(_bits(x), _bits(y)), "lengths = T for every clip differs from the batch without the key"


@gpu
def test_flag_variants_and_reconstruction_ragged(nets, cuda_device):
    dev, lengths, T = cuda_device, [144, 48, 80], 144
    ds_p, _, _, _, _, bm = nets
    for kw in (dict(mask_scheme='full', iter2_cond_noisy_pose=False),
               dict(input_noise=False, mask_scheme='upper', iter2_cond_noisy_traj=False, iter2_cond_noisy_pose=False),
               dict(infill_traj=True, mask_scheme='full', traj_mask_ratio=0.1)):
        lens = [144, 80, 96] if kw.get('infill_traj') else lengths
        args, (vp, vt, tn), seen, pose, traj = _run(nets, dev, lens, T, cond_fn_with_grad=False, **kw)
        assert bool(torch.isfinite(vp).all()) and vp.shape == (3, 294, 1, 143)
        if kw['mask_scheme'] == 'full' and not kw.get('infill_traj'):
            cond0 = seen[0][2]  # round 0: channels >= 22 are zero exactly inside the window, which lies inside the clip
            for b, n in enumerate(lens):
                zero = (cond0[b, 22:290, 0, :n - 1] == 0).all(dim=0).nonzero().flatten()
                assert 1 <= len(zero) <= 30 and int(zero.max()) < n - 1 and int(zero.max() - zero.min()) == len(zero) - 1
        rec = pipeline.reconstruct_outputs(args, ds_p, bm, pose, vp, tn, return_verts=True)
        assert rec['frame_offsets'].tolist() == [0] + torch.tensor(lens).sub(1).cumsum(0).tolist()
        payload = pipeline.result_dict(args, [rec])
        assert ('rec_ric_data_noisy_list' in payload) == bool(args.input_noise)
        for b, n in enumerate(lens):
            assert rec['smpl_verts_rec'][b].shape == (n - 1, 10475, 3) and rec['rec_ric_data_rec_from_abs_traj'][b].shape == (n - 1, 22, 3)
            assert payload['motion_repr_rec_list'][b].shape == (n - 1, 294) and len(payload['motion_repr_rec_list']) == 3
        # the same clips reconstructed alone, from the ragged run's own tensors cut to the clip
        for b, n in enumerate(lens):
            one = {k: v[b:b + 1, ..., :n - 1].contiguous() if v.dim() == 4 else v[b:b + 1, :n - 1].contiguous()
                   for k, v in pose.items() if k != 'lengths'}
            r1 = pipeline.reconstruct_outputs(args, ds_p, bm, one, vp[b:b + 1, ..., :n - 1].contiguous(),
                                              tn[b:b + 1, :n].contiguous(), return_verts=True)
            for key in ('smpl_verts_rec', 'smpl_verts_clean', 'rec_ric_data_rec_from_smpl', 'rec_ric_data_rec_from_abs_traj',
                        'rec_ric_data_clean', 'motion_repr_rec') + (('smpl_verts_noisy', 'motion_repr_noisy') if args.input_noise else ()):
                assert torch.equal(_bits(rec[key][b]), _bits(r1[key][0])), (kw, key, b)


@gpu
def test_refusals_come_before_any_sampling(nets, cuda_device):
    import test_gpu_pipeline as tp
    dev, T = cuda_device, 144
    ds_p, ds_t, mp, mt, mc, bm = nets
    dp, dt, dc = tp._diffusions(dev, 4, pose_respacing="3" + ",0" * 19)

    def call(lengths, grad_type='amass', **kw):
        pose, traj = synthetic.pipeline_batches(2, 5, ds_p, frames=T, device=dev)
        traj['lengths'] = lengths
        seen = []
        with pytest.raises(RohmB200Error):
            pipeline.run_rounds(pipeline.make_args(**kw), mp, mt, mc, dp, dt, dc, ds_p, ds_t, bm, pose, traj,
                                grad_type=grad_type, on_round=lambda *a: seen.append(a))
        assert not seen and 'lengths' not in pose and pose['motion_repr_clean'].shape == (2, T, 294)

    ok = torch.tensor([144, 64], device=dev)
    call(ok, grad_type='prox')
    call(ok, infill_traj=True, traj_mask_ratio=0.1)  # window [65, 79) does not fit 64 frames
    call(torch.tensor([144.0, 64.0], device=dev))
    call(torch.tensor([144, 64, 32], device=dev))
    call(torch.tensor([144, 60], device=dev))
    call(torch.tensor([160, 64], device=dev))
    call(torch.tensor([144, 0], device=dev))
    with pytest.raises(RohmB200Error):
        glue.pose_to_control_cond(torch.zeros(2, 294, 1, 15, device=dev), 16, 272, lengths=glue.device_lengths([15, 16], dev))
    with pytest.raises(RohmB200Error):
        glue.build_pose_cond(torch.zeros(2, 15, 294, device=dev), lengths=torch.tensor([15, 3], device=dev))  # int64
