"""GPU parity tests of the kernels either side of the sampling loops (SURVEY 8f N1-N4): inter-round glue, condition
assembly / occlusion masks, rotation chain edge cases, representation recovery, 2-D reprojection guidance, evaluation loss
dictionaries.  Reference = golden vectors of the unmodified reference (tests/golden/glue.npz, kinematics.npz) and the CPU
oracle at other sizes."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, TOL, golden
from oracle import glue_oracle as go
from oracle import kinematics_oracle as ko
from rohm_b200 import glue, synthetic
from rohm_b200.body_model import BodyModel, kernels_for
from rohm_b200.motion_representation import recover_from_repr_smpl, split_repr
from rohm_b200.posenet import PoseNet
from rohm_b200.trajnet import TrajNet

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def body(cuda_device):
    return BodyModel.create('', device=cuda_device, seed=0), synthetic.smplx_like_model(0)


def _plausible(meta):
    B, T, seed, ds_seed = [int(v) for v in meta]
    ds = synthetic.make_dataset('pose', seed=ds_seed, realistic_std=True)
    return synthetic.plausible_motion(B, T, seed, ds), ds


UNIT = synthetic.make_dataset('pose')  # Mean 0 / Std 1


def test_rotation_chain_edge_cases_through_the_kernel(cuda_device):
    """rot6d -> rotmat -> quaternion -> axis-angle on the reference golden incl. near-identity, exact identity and near-pi
    rotations (the four Shepperd branches and the eps clamps of konia_transform.py:400-443, 616-625)."""
    g = golden("kinematics.npz")
    r6 = torch.from_numpy(g["rot6d_in"]).to(cuda_device)
    aa, R = glue.rot6d_to_angle_axis(r6, want_rotmat=True)
    assert float((R.cpu() - torch.from_numpy(g["rotmat_out"])).abs().max()) < 1e-6
    err = (aa.cpu() - torch.from_numpy(g["aa_out"])).abs().max(dim=1).values
    # generic + near-identity + identity rows: 1e-5; the 8 near-pi rows (ill-conditioned axis) 1e-3
    assert float(err[:-8].max()) < 1e-5, err
    assert float(err[-8:].max()) < 1e-3, err
    # every branch of rotation_matrix_to_quaternion is taken by this input
    Rn = g["rotmat_out"]
    tr = Rn[:, 0, 0] + Rn[:, 1, 1] + Rn[:, 2, 2]
    b1 = (tr <= 0) & (Rn[:, 0, 0] > Rn[:, 1, 1]) & (Rn[:, 0, 0] > Rn[:, 2, 2])
    b2 = (tr <= 0) & ~b1 & (Rn[:, 1, 1] > Rn[:, 2, 2])
    b3 = (tr <= 0) & ~b1 & ~b2
    assert (tr > 0).any() and b1.any() and b2.any() and b3.any()


def test_rotation_chain_edge_cases_through_body_from_repr(body, cuda_device):
    """The same edge rotations as the global orientation / body pose of a representation row, through
    rohm_body_from_repr, against the oracle's SMPL-X joints."""
    bm, model = body
    g = golden("kinematics.npz")
    r6 = torch.from_numpy(g["rot6d_in"])
    n = r6.shape[0]
    T = 8
    B = (n + T - 1) // T
    x = torch.zeros(B, T, 294)
    x[..., 7:13] = torch.tensor([1., 0, 0, 1, 0, 0])
    x[..., 154:280] = torch.tensor([1., 0, 0, 1, 0, 0]).repeat(21)
    flat = x.view(B * T, 294)
    flat[:n, 7:13] = r6                      # edge rotations as global orientation
    flat[:n, 154 + 6 * 4:154 + 6 * 5] = r6.flip(0)  # and as one body joint (5: right knee)
    rep = split_repr(x)
    want = ko.joints_from_smplx(rep, model)
    got = recover_from_repr_smpl({k: v.to(cuda_device) for k, v in rep.items()}, 'smplx_params', bm)
    assert float((got.cpu() - want).abs().max()) < 5e-5


def test_traj_glue_matches_reference_get_repr_smplx(body, cuda_device):
    bm, _ = body
    g = golden("glue.npz")
    x, ds = _plausible(g["repr_meta"])
    clean = x[:, :, 0].permute(0, 2, 1).contiguous()
    sel = [0, 2, 3, 6] + list(range(7, 13)) + list(range(16, 19))
    traj = clean[..., sel].contiguous()
    comp, full = glue.traj_to_full_repr(bm, traj.to(cuda_device), clean.to(cuda_device), ds, UNIT)
    assert torch.equal(comp.cpu(), clean)
    assert float((full.cpu() - torch.from_numpy(g["repr_traj22"]).float()).abs().max()) < 2e-5
    # scatter of the 13 trajectory channels (test_amass_full.py:272-277)
    traj2 = torch.randn(2, 24, 13)
    comp2, _ = glue.traj_to_full_repr(bm, traj2.to(cuda_device), clean.to(cuda_device), ds, UNIT)
    assert torch.equal(comp2.cpu(), go.compose_repr(traj2, clean))


def test_traj_repr_nan_repair_matches_reference(cuda_device):
    """Frame whose forward direction is exactly -y: qbetween gives 0/0 and the reference repairs the first NaN frame with
    its predecessor (motion_representation.py:212-215)."""
    g = golden("glue.npz")
    x, ds = _plausible(g["repr_meta"])
    full = x[:, :, 0].permute(0, 2, 1) * torch.from_numpy(ds.Std) + torch.from_numpy(ds.Mean)
    transl = ko.split_repr(full)['smplx_trans'][0:1]
    dev = cuda_device
    m0, s1 = torch.zeros(294, device=dev), torch.ones(294, device=dev)
    out = glue.traj_repr_from_joints(torch.from_numpy(g["nan_positions"])[None].to(dev),
                                     torch.from_numpy(g["nan_go"])[None].to(dev), transl.to(dev), m0, s1)
    assert bool(torch.isfinite(out).all())
    assert float((out[0].cpu() - torch.from_numpy(g["nan_traj22"]).float()).abs().max()) < 2e-5


@pytest.mark.parametrize("B,T,seed", [(1, 16, 1), (5, 144, 2)])
def test_traj_glue_matches_oracle(body, cuda_device, B, T, seed):
    bm, model = body
    ds_p = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_t = synthetic.make_dataset('traj', seed=4, realistic_std=True)
    clean = synthetic.plausible_motion(B, T, seed, ds_t)[:, :, 0].permute(0, 2, 1).contiguous()
    g = torch.Generator().manual_seed(seed)
    sel = [0, 2, 3, 6] + list(range(7, 13)) + list(range(16, 19))
    traj = clean[..., sel] + 0.05 * torch.randn(B, T, 13, generator=g)
    comp, full = glue.traj_to_full_repr(bm, traj.to(cuda_device), clean.to(cuda_device), ds_t, ds_p)
    comp_o, full_o = go.traj_to_full_repr(traj, clean, ds_t.Mean, ds_t.Std, ds_p.Mean, ds_p.Std, model)
    assert torch.equal(comp.cpu(), comp_o)
    assert float((full.cpu() - full_o).abs().max()) < TOL


def test_control_cond_and_pose_cond_match_oracle(cuda_device):
    g = torch.Generator().manual_seed(5)
    B, Tp = 3, 143
    pose_out = torch.randn(B, 294, 1, Tp, generator=g)
    cc = glue.pose_to_control_cond(pose_out.to(cuda_device), Tp + 1, 272)
    assert torch.equal(cc.cpu(), go.pose_to_control_cond(pose_out, Tp + 1, 272))
    src = torch.randn(B, Tp, 294, generator=g)
    traj_full = torch.randn(B, Tp, 22, generator=g)
    for scheme in ('lower', 'upper', None):
        keep = glue.channel_keep_mask(scheme) if scheme else None
        got = glue.build_pose_cond(src.to(cuda_device), traj_full.to(cuda_device), keep, zero_contact=scheme is not None)
        want = go.build_pose_cond(src, traj_full, scheme, apply_mask=scheme is not None)
        assert torch.equal(got.cpu(), want), scheme
    start, end = torch.tensor([0, 100, 130]), torch.tensor([30, 130, 143])
    got = glue.build_pose_cond(src.to(cuda_device), traj_full.to(cuda_device), None, start, end, zero_contact=True)
    assert torch.equal(got.cpu(), go.build_pose_cond(src, traj_full, 'full', True, start, end))
    # channel-major source (a previous PoseNet output) without trajectory replacement
    got = glue.build_pose_cond(pose_out.to(cuda_device), None, glue.channel_keep_mask('lower'), zero_contact=True)
    want = go.build_pose_cond(pose_out[:, :, 0].permute(0, 2, 1), None, 'lower', True)
    assert torch.equal(got.cpu(), want)


def test_joint_recovery_modes_match_reference(body, cuda_device):
    bm, model = body
    g = golden("glue.npz")
    x, ds = _plausible(g["repr_meta"])
    full = x[:, :, 0].permute(0, 2, 1) * torch.from_numpy(ds.Std) + torch.from_numpy(ds.Mean)
    rep = {k: v.to(cuda_device) for k, v in split_repr(full).items()}
    rel = recover_from_repr_smpl(rep, 'joint_rel_traj', bm)
    assert float((rel.cpu() - torch.from_numpy(g["rel_traj_joints"])).abs().max()) < 2e-5
    ab = recover_from_repr_smpl(rep, 'joint_abs_traj', bm)
    assert float((ab.cpu() - ko.joints_from_abs_traj(ko.split_repr(full))).abs().max()) < 2e-5
    j, v = recover_from_repr_smpl(rep, 'smplx_params', bm, return_verts=True)
    jo, vo = ko.joints_from_smplx(ko.split_repr(full), model, return_verts=True)
    assert j.shape == (2, 24, 22, 3) and v.shape == (2, 24, 10475, 3)
    assert float((j.cpu() - jo).abs().max()) < 2e-5 and float((v.cpu() - vo).abs().max()) < TOL
    assert float((j.cpu() - torch.from_numpy(g["repr_joints"])).abs().max()) < 2e-5
    with pytest.raises(Exception):
        recover_from_repr_smpl(rep, 'smplx_params', bm, return_full_joints=True)


def test_from_repr_with_vertices_both_layouts(body, cuda_device):
    """rohm_body_from_repr with vertices, channel-major and channels-last inputs."""
    bm, model = body
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    x = synthetic.plausible_motion(2, 9, 17, ds)
    mean, std = glue.stats_on(ds, cuda_device)
    k = kernels_for(bm, cuda_device, 18, with_vertices=True)
    j1, v1 = k.from_repr(x.to(cuda_device), mean, std, want_vertices=True)
    xl = x[:, :, 0].permute(0, 2, 1).contiguous()
    j2, v2 = k.from_repr(xl.to(cuda_device), mean, std, want_vertices=True, channels_last=True)
    assert torch.equal(j1, j2) and torch.equal(v1, v2)
    full = xl * torch.from_numpy(ds.Std) + torch.from_numpy(ds.Mean)
    jo, vo = ko.joints_from_smplx(ko.split_repr(full), model, return_verts=True)
    assert float((v1.cpu() - vo).abs().max()) < TOL


def test_dense_skinning_fallback_matches_sparse():
    """skin_dense_kernel (models with more than 8 bones per vertex) forced through ROHM_B200_DENSE_SKIN=1 in a fresh
    process; must agree with the oracle like the sparse kernel does."""
    code = (
        "import torch, sys\n"
        f"sys.path.insert(0, {ROOT!r})\n"
        "from rohm_b200 import synthetic\n"
        "from rohm_b200.body_model import BodyModel\n"
        "from oracle import kinematics_oracle as ko\n"
        "dev = torch.device('cuda:0')\n"
        "bm = BodyModel.create('', device=dev)\n"
        "g = torch.Generator().manual_seed(3)\n"
        "N = 147\n"
        "go, bp, be, tr = 0.3*torch.randn(N,3,generator=g), 0.3*torch.randn(N,63,generator=g), torch.randn(N,10,generator=g), torch.randn(N,3,generator=g)\n"
        "out = bm(transl=tr.to(dev), global_orient=go.to(dev), body_pose=bp.to(dev), betas=be.to(dev))\n"
        "j, v = ko.smplx_forward(synthetic.smplx_like_model(0), go, bp, be, tr, return_verts=True, dtype=torch.float64)\n"
        "err = float((out.vertices.cpu().double() - v).abs().max())\n"
        "print('dense skin err', err)\n"
        "assert err < 5e-5, err\n")
    # the fused blend + skinning launch takes precedence over both skin kernels: switch it off to reach them.  First the dense
    # fallback, then the sparse two-kernel path (blend GEMM -> v_posed -> skin_kernel), the fallback for models whose 32-vertex
    # tiles touch more than 16 bones.
    for extra in ({"ROHM_B200_DENSE_SKIN": "1"}, {}):
        env = dict(os.environ, ROHM_B200_FUSED_LBS="0", **extra)
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "dense skin err" in r.stdout


def test_body_model_rejects_nonzero_hand_pose(body, cuda_device):
    bm, _ = body
    z = lambda *s: torch.zeros(*s, device=cuda_device)
    with pytest.raises(Exception):
        bm(transl=z(2, 3), global_orient=z(2, 3), body_pose=z(2, 63), betas=z(2, 10),
           left_hand_pose=torch.ones(2, 45, device=cuda_device))


def _posenet(cuda_device, ds):
    m = PoseNet(dataset=ds, body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4,
                device=cuda_device, traj_feat_dim=22)
    m.load_state_dict({k: v.cpu() for k, v in synthetic.synth_state_dict(m, 1).items()})
    return m.to(cuda_device).eval()


def test_projection_guidance_matches_reference_autograd(cuda_device):
    """guide_2d_projection_with_smpl: analytic CUDA VJP through the 22-joint tree vs the reference's autograd."""
    g = golden("glue.npz")
    x, ds = _plausible(g["repr_meta"])
    dev = cuda_device
    ds.cam_R, ds.cam_t = torch.from_numpy(g["proj_cam_R"]).to(dev), torch.from_numpy(g["proj_cam_t"]).to(dev)
    m = _posenet(dev, ds)
    t = lambda k: torch.from_numpy(g[k]).to(dev)
    batch = {'transf_matrix': t("proj_transf"), 'focal_length': t("proj_focal"), 'camera_center': t("proj_center"),
             'keypoints_2d': t("proj_kp")}
    xg = x.to(dev)
    grad = m.guide_2d_projection_with_smpl(batch, {'pred_xstart': xg}, None, compute_grad='x_0').cpu()
    ref = torch.from_numpy(g["proj_grad"])
    scale = float(ref.abs().max())
    err = float((grad - ref).abs().max())
    print(f"projection guidance: max |cuda - reference autograd| = {err:.3e} (gradient scale {scale:.3e})")
    assert err < 2e-4 * scale
    assert float(grad[:, :22].abs().max()) == 0.0 and float(grad[:, -4:].abs().max()) == 0.0


@pytest.mark.parametrize("B,T,seed", [(1, 3, 1), (4, 143, 2)])
def test_projection_guidance_matches_oracle_autograd(cuda_device, B, T, seed):
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    x = synthetic.plausible_motion(B, T, seed, ds)
    g = torch.Generator().manual_seed(seed)
    cam_R = torch.tensor([[1., 0, 0], [0, 0, 1], [0, -1, 0]])
    cam_t = torch.tensor([[0.2, -5.0, 1.0]])
    tm = torch.eye(4).repeat(B, 1, 1)
    tm[:, :3, 3] = 0.1 * torch.randn(B, 3, generator=g)
    focal, center = torch.tensor([[1000., 990.]]).repeat(B, 1), torch.tensor([[900., 500.]]).repeat(B, 1)
    kp = torch.cat([900 + 300 * torch.randn(B, T, 22, 1, generator=g), 500 + 200 * torch.randn(B, T, 22, 1, generator=g),
                    torch.rand(B, T, 22, 1, generator=g)], dim=-1)
    ref, _ = go.guide_projection(x.double(), torch.from_numpy(ds.Mean).double(), torch.from_numpy(ds.Std).double(),
                                 synthetic.smplx_like_model(0), tm.double(), cam_R.double(), cam_t.double(), focal.double(),
                                 center.double(), kp.double())
    dev = cuda_device
    ds.cam_R, ds.cam_t = cam_R.to(dev), cam_t.to(dev)
    m = _posenet(dev, ds)
    batch = {'transf_matrix': tm.to(dev), 'focal_length': focal.to(dev), 'camera_center': center.to(dev),
             'keypoints_2d': kp.to(dev)}
    xg = x.to(dev)
    grad = m.guide_2d_projection_with_smpl(batch, {'pred_xstart': xg}, None, compute_grad='x_0').cpu().double()
    scale = float(ref.abs().max())
    assert scale > 0 and float((grad - ref).abs().max()) < 2e-4 * scale


def _check_losses(got, names, values, rtol=2e-4):
    assert list(got.keys()) == [str(n) for n in names]
    for n, v in zip(names, values):
        a = float(got[str(n)])
        if np.isnan(v):
            assert np.isnan(a), n
        else:
            assert abs(a - v) <= rtol * max(abs(v), 1e-6) + 1e-9, (str(n), a, v)


def test_eval_loss_dictionaries_match_reference(body, cuda_device):
    """compute_losses_with_smpl of both models (the default compute_loss=True path of eval_losses) vs the reference."""
    bm, _ = body
    g = golden("glue.npz")
    x, ds = _plausible(g["repr_meta"])
    dev = cuda_device
    m = _posenet(dev, ds)
    rec = torch.from_numpy(g["pose_loss_rec"]).to(dev)
    got = m.compute_losses_with_smpl({'motion_repr_clean': x.to(dev)}, rec, smplx_model=bm, epoch=0)
    _check_losses(got, g["pose_loss_names"], g["pose_loss_values"])
    dst = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    mt = TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=False, device=dev, dataset=dst,
                 repr_abs_only=True).to(dev).eval()
    clean_cl = x[:, :, 0].permute(0, 2, 1).contiguous().to(dev)
    got = mt.compute_losses_with_smpl({'motion_repr_clean': clean_cl}, torch.from_numpy(g["traj_loss_rec"]).to(dev),
                                      smplx_model=bm)
    _check_losses(got, g["traj_loss_names"], g["traj_loss_values"])


def test_fused_lbs_falls_back_when_a_tile_touches_too_many_bones(cuda_device):
    """The fused blend + skinning launch needs at most 16 distinct bones per 32 consecutive vertices.  A body model whose
    vertices are in random order breaks that: the handle must choose the two-kernel path by itself and stay correct; the
    body-part-ordered model takes the fused path."""
    t = synthetic.smplx_like_model(0)
    V = t['v_template'].shape[0]
    perm = torch.randperm(V, generator=torch.Generator().manual_seed(5))
    shuffled = dict(t)
    shuffled['v_template'], shuffled['shapedirs'] = t['v_template'][perm], t['shapedirs'][perm]
    shuffled['lbs_weights'], shuffled['J_regressor'] = t['lbs_weights'][perm], t['J_regressor'][:, perm]
    shuffled['posedirs'] = t['posedirs'].view(-1, V, 3)[:, perm].reshape(-1, V * 3)
    g = torch.Generator().manual_seed(9)
    N = 40
    gor, bp = 0.3 * torch.randn(N, 3, generator=g), 0.3 * torch.randn(N, 63, generator=g)
    be, tr = torch.randn(N, 10, generator=g), torch.randn(N, 3, generator=g)
    for tensors, fused in ((shuffled, 0), (t, 1)):
        bm = BodyModel(tensors).to(cuda_device)
        out = bm(transl=tr.to(cuda_device), global_orient=gor.to(cuda_device), body_pose=bp.to(cuda_device), betas=be.to(cuda_device))
        k = kernels_for(bm, cuda_device, N, with_vertices=True)
        assert k.lib.rohm_body_uses_fused_lbs(k.handle) == fused
        _, v = ko.smplx_forward(tensors, gor, bp, be, tr, return_verts=True, dtype=torch.float64)
        assert float((out.vertices.cpu().double() - v).abs().max()) < 5e-5
