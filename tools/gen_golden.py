"""Generates tests/golden/*.npz by running the UNMODIFIED reference (sanweiliti/RoHM mounted at /root/reference) on
seeded synthetic weights and inputs.  Run in the build container only (the reference does not travel to the GPU box):

    python tools/gen_golden.py

Everything needed to regenerate an input is a seed: weights come from rohm_b200.synthetic.synth_state_dict, inputs
from torch.Generator streams.  The only stand-in is the third-party ``smplx`` package (absent, licence-gated model):
``smplx.create`` returns the oracle's SMPL-X restatement on the synthetic body model, so the reference code around
the body-model call (rot6d -> axis-angle, losses, autograd) is the real thing.
"""
import argparse
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.dont_write_bytecode = True
sys.path.insert(0, ROOT)
sys.path.append('/root/reference')  # AFTER the repo: only used for the reference's own top-level packages below

import numpy as np
import torch
import torch.nn as nn
from scipy.spatial.transform import Rotation as ref_rotation

from oracle import kinematics_oracle as ko
from rohm_b200 import synthetic

OUT = os.path.join(ROOT, "tests", "golden")


class _StubBody(nn.Module):
    """smplx stand-in: same call signature / output attributes, arithmetic = oracle restatement."""

    def __init__(self):
        super().__init__()
        self.model = synthetic.smplx_like_model(0)

    def forward(self, transl=None, global_orient=None, body_pose=None, betas=None, **unused):
        joints, verts = ko.smplx_forward(self.model, global_orient, body_pose, betas, transl, return_verts=False)
        return types.SimpleNamespace(joints=joints, vertices=verts)


def import_reference():
    stub = types.ModuleType('smplx')
    stub.create = lambda **kw: _StubBody()
    sys.modules['smplx'] = stub
    # make sure the reference's namespace packages win for these imports
    for name in ("model", "diffusion", "utils", "data_loaders"):
        sys.modules.pop(name, None)
    sys.path.insert(0, '/root/reference')
    import diffusion.gaussian_diffusion_posenet as gdp
    import diffusion.gaussian_diffusion_trajnet as gdt
    import diffusion.respace as respace
    import utils.model_util as model_util
    import model.posenet as ref_posenet
    import model.trajnet as ref_trajnet
    import data_loaders.motion_representation as mr
    import data_loaders.common.quaternion as quat
    import utils.konia_transform as kt
    import utils.other_utils as ou
    sys.path.pop(0)
    return types.SimpleNamespace(gdp=gdp, gdt=gdt, respace=respace, model_util=model_util, posenet=ref_posenet,
                                 trajnet=ref_trajnet, mr=mr, quat=quat, kt=kt, ou=ou)


TABLES = ("betas", "alphas_cumprod", "alphas_cumprod_prev", "alphas_cumprod_next", "sqrt_alphas_cumprod",
          "sqrt_one_minus_alphas_cumprod", "log_one_minus_alphas_cumprod", "sqrt_recip_alphas_cumprod",
          "sqrt_recipm1_alphas_cumprod", "posterior_variance", "posterior_log_variance_clipped",
          "posterior_mean_coef1", "posterior_mean_coef2")


def gen_schedules(ref):
    out = {}
    cases = [("cosine", 1000, ''), ("cosine", 100, ''), ("cosine", 50, ''), ("cosine", 1000, 'ddim100'),
             ("cosine", 1000, '100'), ("cosine", 1000, 'ddim50'), ("cosine", 300, '10,15,20'), ("linear", 100, ''),
             ("linear", 1000, 'ddim20')]
    for idx, (sched, steps, resp) in enumerate(cases):
        args = argparse.Namespace(noise_schedule=sched, sigma_small=True)
        d = ref.model_util.create_gaussian_diffusion(args, gd=ref.gdp, return_class=ref.respace.SpacedDiffusionPoseNet,
                                                     num_diffusion_timesteps=steps, timestep_respacing=resp, device='cpu')
        out[f"c{idx}_meta"] = np.array([sched, str(steps), resp])
        out[f"c{idx}_timestep_map"] = np.array(d.timestep_map, dtype=np.int64)
        for t in TABLES:
            out[f"c{idx}_{t}"] = getattr(d, t)
    out["n_cases"] = np.array(len(cases))
    # space_timesteps known answers
    out["space_300_10_15_20"] = np.array(sorted(ref.respace.space_timesteps(300, [10, 15, 20])), dtype=np.int64)
    out["space_1000_ddim100"] = np.array(sorted(ref.respace.space_timesteps(1000, "ddim100")), dtype=np.int64)
    out["space_1000_100"] = np.array(sorted(ref.respace.space_timesteps(1000, "100")), dtype=np.int64)
    out["space_1000_7_13_29"] = np.array(sorted(ref.respace.space_timesteps(1000, "7,13,29")), dtype=np.int64)
    try:
        ref.respace.space_timesteps(1000, "ddim300")
        out["ddim300_raises"] = np.array(0)
    except ValueError:
        out["ddim300_raises"] = np.array(1)
    np.savez_compressed(os.path.join(OUT, "schedules.npz"), **out)
    print("schedules.npz", len(out), "arrays")


def build_ref_posenet(ref, seed, device='cpu'):
    ds = synthetic.make_dataset('pose')
    m = ref.posenet.PoseNet(dataset=ds, body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4,
                            dropout=0.1, activation="gelu", body_model_path='', device=device, traj_feat_dim=22)
    sd = synthetic.synth_state_dict(m, seed)
    m.load_state_dict(sd)
    return m.eval(), sd


def build_ref_trajnet(ref, seed, control):
    ds = synthetic.make_dataset('traj')
    m = ref.trajnet.TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=control, device='cpu',
                            dataset=ds, repr_abs_only=True)
    sd = synthetic.synth_state_dict(m, seed)
    m.load_state_dict(sd)
    return m.eval(), sd


def gen_posenet(ref):
    out = {}
    m, _ = build_ref_posenet(ref, seed=1)
    for idx, (B, T, s) in enumerate([(2, 16, 11), (1, 8, 12), (1, 143, 13)]):
        g = torch.Generator().manual_seed(s)
        x = torch.randn(B, 294, 1, T, generator=g)
        cond = synthetic.posenet_batch(B, T, s + 100)['cond']
        ts = torch.randint(0, 1000, (B,), generator=g)
        with torch.no_grad():
            y = m({'x_t': x, 'cond': cond}, ts)
        out[f"c{idx}_meta"] = np.array([B, T, s])
        out[f"c{idx}_timesteps"] = ts.numpy()
        out[f"c{idx}_out"] = y.numpy()
    out["n_cases"] = np.array(3)
    out["weight_seed"] = np.array(1)
    np.savez_compressed(os.path.join(OUT, "posenet_forward.npz"), **out)
    print("posenet_forward.npz")


def gen_trajnet(ref):
    out = {}
    idx = 0
    for control in (False, True):
        m, _ = build_ref_trajnet(ref, seed=2, control=control)
        for (B, T, s) in [(2, 32, 21), (1, 144, 22)]:
            g = torch.Generator().manual_seed(s)
            x = torch.randn(B, T, 13, generator=g)
            batch = synthetic.trajnet_batch(B, T, s + 100, control=control)
            batch['x_t'] = x
            ts = torch.randint(0, 100, (B,), generator=g)
            with torch.no_grad():
                y = m(batch, ts)
            out[f"c{idx}_meta"] = np.array([B, T, s, int(control)])
            out[f"c{idx}_timesteps"] = ts.numpy()
            out[f"c{idx}_out"] = y.numpy()
            idx += 1
    out["n_cases"] = np.array(idx)
    out["weight_seed"] = np.array(2)
    np.savez_compressed(os.path.join(OUT, "trajnet_forward.npz"), **out)
    print("trajnet_forward.npz")


class _NoiseTape:
    """A stand-in for the ``th`` name inside a reference diffusion module: forwards everything to torch except
    randn / randn_like, which draw from a seeded CPU stream (so the oracle and the CUDA path can replay it)."""

    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)

    def randn(self, *shape, device=None, **kw):
        return torch.randn(*shape, generator=self.g)

    def randn_like(self, x):
        return torch.randn(x.shape, generator=self.g)

    def __getattr__(self, name):
        return getattr(torch, name)


class _patched_th:
    def __init__(self, module, seed):
        self.module, self.tape = module, _NoiseTape(seed)

    def __enter__(self):
        self.real = self.module.th
        self.module.th = self.tape

    def __exit__(self, *a):
        self.module.th = self.real


def gen_sampling(ref):
    out = {}
    # (a) BASELINE config 1: TrajNet vanilla, 1 clip of 144 frames, 50 DDPM steps, through eval_losses
    m, _ = build_ref_trajnet(ref, seed=2, control=False)
    args = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    d = ref.model_util.create_gaussian_diffusion(args, gd=ref.gdt, return_class=ref.respace.SpacedDiffusionTrajNet,
                                                 num_diffusion_timesteps=50, timestep_respacing='', device='cpu')
    batch = synthetic.trajnet_batch(1, 144, 31)
    with _patched_th(ref.gdt, 41), torch.no_grad():
        _, y = d.eval_losses(model=m, batch=batch, shape=[1, 144, 13], progress=False, clip_denoised=False,
                             timestep_respacing='', cond_fn_with_grad=True, compute_loss=False, smplx_model=None)
    out["traj50_out"] = y.numpy()
    out["traj50_meta"] = np.array([1, 144, 31, 41, 50])

    # (b) PoseNet, respaced ancestral sampling ('ddim20' retained steps of a 1000-step base), 1 clip x 16 frames
    mp, _ = build_ref_posenet(ref, seed=1)
    dp = ref.model_util.create_gaussian_diffusion(args, gd=ref.gdp, return_class=ref.respace.SpacedDiffusionPoseNet,
                                                  num_diffusion_timesteps=1000, timestep_respacing='ddim20', device='cpu')
    batch = synthetic.posenet_batch(1, 16, 32)
    with _patched_th(ref.gdp, 42), torch.no_grad():
        y = dp.p_sample_loop(mp, batch, [1, 294, 1, 16], clip_denoised=False, cond_fn_with_grad=False)
    out["pose_ddim20_out"] = y.numpy()
    out["pose_ddim20_meta"] = np.array([1, 16, 32, 42, 20])

    # (c) PoseNet guided sampling (p_sample_with_grad, grad_type='amass') in the regime the guidance weights were
    #     tuned for: the last 12 steps of the 1000-step chain (skip_timesteps=988 -> t = 11..0, all guided), started
    #     from q_sample(init_image = a plausible motion).
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    mp.dataset = ds
    mp.device = 'cpu'
    dg = ref.model_util.create_gaussian_diffusion(args, gd=ref.gdp, return_class=ref.respace.SpacedDiffusionPoseNet,
                                                  num_diffusion_timesteps=1000, timestep_respacing='', device='cpu')
    init = synthetic.plausible_motion(2, 12, 33, ds)
    batch = {'cond': init.clone()}
    traj = []
    with _patched_th(ref.gdp, 43):
        for o in dg.p_sample_loop_progressive(mp, batch, [2, 294, 1, 12], clip_denoised=False, cond_fn_with_grad=True,
                                              grad_type='amass', skip_timesteps=994, init_image=init):
            traj.append((o['x_t'].detach().clone(), o['pred_xstart'].detach().clone(), o['sample'].detach().clone()))
    # The guided chain is ill-conditioned (weight 3e6 on a loss with hard masks; the reference README says results
    # are not reproducible across machines), so the fixture stores every step for teacher-forced comparison.
    out["pose_guided_xt"] = torch.stack([t[0] for t in traj]).numpy()
    out["pose_guided_x0"] = torch.stack([t[1] for t in traj]).numpy()
    out["pose_guided_sample"] = torch.stack([t[2] for t in traj]).numpy()
    out["pose_guided_meta"] = np.array([2, 12, 33, 43, 994])
    np.savez_compressed(os.path.join(OUT, "sampling.npz"), **out)
    print("sampling.npz")


def gen_kinematics(ref):
    out = {}
    g = torch.Generator().manual_seed(51)
    # rotations: generic, near identity, near pi, exactly identity
    r6 = torch.randn(64, 6, generator=g)
    near_id = torch.tensor([1., 0, 0, 1, 0, 0]).repeat(8, 1) + 1e-4 * torch.randn(8, 6, generator=g)
    ident = torch.tensor([[1., 0, 0, 1, 0, 0]])
    # rotation by ~pi about random axes, given as 6d (first two columns, row-major 3x2)
    ax = torch.nn.functional.normalize(torch.randn(8, 3, generator=g), dim=1)
    ang = (np.pi - 1e-3 * torch.rand(8, generator=g))
    K = torch.zeros(8, 3, 3)
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 0], K[:, 1, 2], K[:, 2, 0], K[:, 2, 1] = -ax[:, 2], ax[:, 1], ax[:, 2], -ax[:, 0], -ax[:, 1], ax[:, 0]
    Rpi = torch.eye(3) + torch.sin(ang)[:, None, None] * K + (1 - torch.cos(ang))[:, None, None] * (K @ K)
    r6 = torch.cat([r6, near_id, ident, Rpi[:, :, :2].reshape(8, 6)], dim=0)
    R = ref.quat.rot6d_to_rotmat(r6)
    aa = ref.kt.rotation_matrix_to_angle_axis(R)
    out["rot6d_in"], out["rotmat_out"], out["aa_out"] = r6.numpy(), R.numpy(), aa.numpy()

    # joint_abs_traj recovery and the skating guidance gradient on a plausible motion
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    x = synthetic.plausible_motion(2, 12, 52, ds)  # [2,294,1,12]
    full = x[:, :, 0].permute(0, 2, 1) * torch.from_numpy(ds.Std) + torch.from_numpy(ds.Mean)
    rep, cur = {}, 0
    for name in ko.REPR_LIST:
        rep[name] = full[..., cur:cur + ko.REPR_DIM_DICT[name]]
        cur += ko.REPR_DIM_DICT[name]
    body = _StubBody()
    out["abs_traj_joints"] = ref.mr.recover_from_repr_smpl(rep, recover_mode='joint_abs_traj', smplx_model=body).numpy()
    out["smplx_joints"] = ref.mr.recover_from_repr_smpl(rep, recover_mode='smplx_params', smplx_model=body).numpy()
    m, _ = build_ref_posenet(ref, seed=1)
    m.dataset, m.device = ds, 'cpu'
    grad = m.guide_skating_with_smpl({'x_t': x}, {'pred_xstart': x}, None, compute_grad='x_0')
    out["skating_grad"] = grad.detach().numpy()
    out["kin_meta"] = np.array([2, 12, 52, 3])
    np.savez_compressed(os.path.join(OUT, "kinematics.npz"), **out)
    print("kinematics.npz  grad absmax", float(grad.abs().max()))


def _rep_dict(full):
    rep, cur = {}, 0
    for name in ko.REPR_LIST:
        rep[name] = full[..., cur:cur + ko.REPR_DIM_DICT[name]]
        cur += ko.REPR_DIM_DICT[name]
    return rep


def gen_glue(ref):
    """Driver-side functions around the loops: get_repr_smplx (trajectory block), 'joint_rel_traj' recovery, the two
    compute_losses_with_smpl dictionaries and the 2-D reprojection guidance gradient (reference autograd)."""
    out = {}
    body = _StubBody()
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    # (a) get_repr_smplx on SMPL-X joints of a plausible motion, 2 clips x 24 frames (+ a clip that faces -y at one frame so
    #     the NaN repair of motion_representation.py:212-215 is exercised)
    x = synthetic.plausible_motion(2, 24, 61, ds)
    full = x[:, :, 0].permute(0, 2, 1) * torch.from_numpy(ds.Std) + torch.from_numpy(ds.Mean)
    rep = _rep_dict(full)
    joints = ref.mr.recover_from_repr_smpl(rep, recover_mode='smplx_params', smplx_model=body).numpy()
    traj = []
    for i in range(2):
        go = ref.kt.rotation_matrix_to_angle_axis(ref.quat.rot6d_to_rotmat(rep['smplx_rot_6d'][i]))
        bp = ref.kt.rotation_matrix_to_angle_axis(ref.quat.rot6d_to_rotmat(rep['smplx_body_pose_6d'][i].reshape(-1, 6)))
        params = {'transl': rep['smplx_trans'][i].numpy(), 'global_orient': go.numpy(),
                  'body_pose': bp.reshape(-1, 63).numpy(), 'betas': rep['smplx_betas'][i].numpy()}
        d = ref.mr.get_repr_smplx(positions=joints[i], smplx_params_dict=params, feet_vel_thre=5e-5)
        traj.append(np.concatenate([d[k] for k in ko.REPR_LIST], axis=-1)[:, 0:22])
    out["repr_x"] = x.numpy()
    out["repr_joints"] = joints
    out["repr_traj22"] = np.asarray(traj)
    out["repr_meta"] = np.array([2, 24, 61, 3])
    # NaN repair: hips/shoulders arranged so that the forward direction is exactly -y at frame 5
    pos = joints[0].copy()
    pos[5, 1], pos[5, 2], pos[5, 17], pos[5, 16] = [0, 0, 0], [1, 0, 0], [0, 0, 0], [1, 0, 0]
    go0 = ref.kt.rotation_matrix_to_angle_axis(ref.quat.rot6d_to_rotmat(rep['smplx_rot_6d'][0])).numpy()
    params = {'transl': rep['smplx_trans'][0].numpy(), 'global_orient': go0,
              'body_pose': np.zeros((24, 63), np.float32), 'betas': rep['smplx_betas'][0].numpy()}
    d = ref.mr.get_repr_smplx(positions=pos, smplx_params_dict=params, feet_vel_thre=5e-5)
    out["nan_positions"], out["nan_go"] = pos, go0
    out["nan_traj22"] = np.concatenate([d[k] for k in ko.REPR_LIST], axis=-1)[:, 0:22]
    # (b) joint_rel_traj recovery
    out["rel_traj_joints"] = ref.mr.recover_from_repr_smpl(rep, recover_mode='joint_rel_traj', smplx_model=body).numpy()
    # (c) evaluation loss dictionaries
    mp, _ = build_ref_posenet(ref, seed=1)
    mp.dataset, mp.device = ds, 'cpu'
    g = torch.Generator().manual_seed(62)
    rec = x + 0.05 * torch.randn(x.shape, generator=g)
    ld = mp.compute_losses_with_smpl({'motion_repr_clean': x}, rec, smplx_model=body, epoch=0)
    out["pose_loss_names"] = np.array(list(ld.keys()))
    out["pose_loss_values"] = np.array([float(v) for v in ld.values()], dtype=np.float64)
    out["pose_loss_rec"] = rec.numpy()
    dst = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    mt, _ = build_ref_trajnet(ref, seed=2, control=False)
    mt.dataset, mt.device = dst, 'cpu'
    clean_cl = x[:, :, 0].permute(0, 2, 1).contiguous()
    traj_rec = torch.cat([clean_cl[..., 0:1], clean_cl[..., 2:4], clean_cl[..., 6:7], clean_cl[..., 7:13],
                          clean_cl[..., 16:19]], dim=-1) + 0.05 * torch.randn(2, 24, 13, generator=g)
    ld = mt.compute_losses_with_smpl({'motion_repr_clean': clean_cl}, traj_rec, smplx_model=body)
    out["traj_loss_names"] = np.array(list(ld.keys()))
    out["traj_loss_values"] = np.array([float(v) for v in ld.values()], dtype=np.float64)
    out["traj_loss_rec"] = traj_rec.numpy()
    # (d) 2-D reprojection guidance (autograd through the reference code + stub body)
    B, T = 2, 24
    cam2world = torch.eye(4)
    ang = 0.3
    cam2world[:3, :3] = torch.tensor([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]]).float() @ \
        torch.tensor([[1., 0, 0], [0, 0, 1], [0, -1, 0]])
    cam2world[:3, 3] = torch.tensor([0.3, -4.0, 1.2])
    ds.cam_R, ds.cam_t = cam2world[:3, :3].reshape(3, 3).float(), cam2world[:3, 3].reshape(1, 3).float()
    tm = torch.eye(4).repeat(B, 1, 1)
    for b in range(B):
        a = 0.4 * (b + 1)
        tm[b, :3, :3] = torch.tensor([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]).float()
        tm[b, :3, 3] = torch.tensor([0.1 * b, -0.2, 0.05])
    batch = {'x_t': x, 'transf_matrix': tm.float(), 'focal_length': torch.tensor([[1060.0, 1058.0]]).repeat(B, 1),
             'camera_center': torch.tensor([[951.0, 536.0]]).repeat(B, 1)}
    kp = torch.zeros(B, T + 2, 22, 3)
    kp[..., 0] = 951.0 + 300.0 * torch.randn(B, T + 2, 22, generator=g)
    kp[..., 1] = 536.0 + 200.0 * torch.randn(B, T + 2, 22, generator=g)
    kp[..., 2] = (torch.rand(B, T + 2, 22, generator=g) > 0.3).float() * torch.rand(B, T + 2, 22, generator=g)
    batch['keypoints_2d'] = kp
    gr = mp.guide_2d_projection_with_smpl(batch, {'pred_xstart': x}, None, compute_grad='x_0')
    out["proj_grad"] = gr.detach().numpy()
    out["proj_cam_R"], out["proj_cam_t"] = ds.cam_R.numpy(), ds.cam_t.numpy()
    out["proj_transf"], out["proj_focal"], out["proj_center"] = tm.numpy(), batch['focal_length'].numpy(), batch['camera_center'].numpy()
    out["proj_kp"] = kp.numpy()
    np.savez_compressed(os.path.join(OUT, "glue.npz"), **out)
    print("glue.npz  proj grad absmax", float(gr.abs().max()), " nan-repair traj finite:", bool(np.isfinite(out["nan_traj22"]).all()))


def gen_clip_guidance(ref):
    """Per-clip guidance normalisers: the reference's guide_skating_with_smpl and guide_2d_projection_with_smpl on each clip
    of a padded batch run alone, as a one-clip batch of its own frames.  Clip 2 has one frame and clip 3 no foot in
    contact, so nothing of either skates (the reference returns a 0-dim zero, stored as a zero gradient)."""
    out = {}
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    lengths = [24, 13, 1, 17]
    B, T = len(lengths), 24
    x = synthetic.plausible_motion(B, T, 71, ds)
    mean, std = torch.from_numpy(ds.Mean), torch.from_numpy(ds.Std)
    x[3, -4:] = ((0.0 - mean[-4:]) / std[-4:]).reshape(4, 1, 1)  # contact labels 0: no skating pair in clip 3
    for b, n in enumerate(lengths):
        x[b, ..., n:] = float("nan")  # never read by a per-clip computation
    g = torch.Generator().manual_seed(72)
    cam2world = torch.eye(4)
    ang = -0.2
    cam2world[:3, :3] = torch.tensor([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]]).float() @ \
        torch.tensor([[1., 0, 0], [0, 0, 1], [0, -1, 0]])
    cam2world[:3, 3] = torch.tensor([-0.2, -3.5, 1.1])
    ds.cam_R, ds.cam_t = cam2world[:3, :3].reshape(3, 3).float(), cam2world[:3, 3].reshape(1, 3).float()
    tm = torch.eye(4).repeat(B, 1, 1)
    for b in range(B):
        a = -0.3 * (b + 1)
        tm[b, :3, :3] = torch.tensor([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]).float()
        tm[b, :3, 3] = torch.tensor([0.05 * b, 0.1, -0.02 * b])
    focal = torch.tensor([[1060.0, 1058.0]]).repeat(B, 1) + torch.arange(B).float()[:, None]
    center = torch.tensor([[951.0, 536.0]]).repeat(B, 1) - torch.arange(B).float()[:, None]
    kp = torch.zeros(B, T + 3, 22, 3)
    kp[..., 0] = 951.0 + 300.0 * torch.randn(B, T + 3, 22, generator=g)
    kp[..., 1] = 536.0 + 200.0 * torch.randn(B, T + 3, 22, generator=g)
    kp[..., 2] = (torch.rand(B, T + 3, 22, generator=g) > 0.3).float() * torch.rand(B, T + 3, 22, generator=g)
    mp, _ = build_ref_posenet(ref, seed=1)
    mp.dataset, mp.device = ds, 'cpu'
    skating, proj, proj_loss, skates = np.zeros((B, 294, 1, T), np.float32), np.zeros((B, 294, 1, T), np.float32), [], []
    for b, n in enumerate(lengths):
        xb = x[b:b + 1, ..., :n].contiguous()
        gs = mp.guide_skating_with_smpl({'x_t': xb}, {'pred_xstart': xb}, None, compute_grad='x_0')
        skates.append(int(gs.dim() > 0))
        if gs.dim() > 0:
            skating[b:b + 1, ..., :n] = gs.detach().numpy()
        batch = {'x_t': xb, 'transf_matrix': tm[b:b + 1].float(), 'focal_length': focal[b:b + 1],
                 'camera_center': center[b:b + 1], 'keypoints_2d': kp[b:b + 1]}
        gp = mp.guide_2d_projection_with_smpl(batch, {'pred_xstart': xb}, None, compute_grad='x_0')
        proj[b:b + 1, ..., :n] = gp.detach().numpy()
    out["x"], out["lengths"], out["skates"] = x.numpy(), np.array(lengths, np.int64), np.array(skates, np.int64)
    out["ds_seed"] = np.array(3)
    out["skating_grad"], out["proj_grad"] = skating, proj
    out["cam_R"], out["cam_t"] = ds.cam_R.numpy(), ds.cam_t.numpy()
    out["transf"], out["focal"], out["center"], out["kp"] = tm.numpy(), focal.numpy(), center.numpy(), kp.numpy()
    np.savez_compressed(os.path.join(OUT, "clip_guidance.npz"), **out)
    print("clip_guidance.npz  skates per clip", skates, " skating absmax", float(np.abs(skating).max()),
          " proj absmax", float(np.abs(proj).max()))


POSE_RESPACING = "12" + ",0" * 19
POSE_RECORDED_STEPS = (6, 5, 1, 0)


def gen_pipeline(ref):
    """BASELINE config 4 in miniature, driven through the UNMODIFIED reference: the call sequence of
    test_amass_full.py:231-384 (TrajNet -> host glue -> PoseNet with in-loop skating guidance, 2 rounds, round 2 through
    TrajControl) on 2 clips x 144 frames with 10-step TrajNet and 12-step PoseNet schedules (every PoseNet step guided)."""
    get_repr_smplx = ref.mr.get_repr_smplx
    out = {}
    B, Tn_steps, Pn_steps, rounds = 2, 10, 12, 2
    ds_pose = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_traj = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    body = _StubBody()
    mp, _ = build_ref_posenet(ref, seed=1)
    mp.dataset, mp.device = ds_pose, 'cpu'
    mt, _ = build_ref_trajnet(ref, seed=2, control=False)
    mc, _ = build_ref_trajnet(ref, seed=4, control=True)
    args = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    mk = ref.model_util.create_gaussian_diffusion
    # PoseNet: the last 50 steps of the 1000-step schedule thinned to 12 (respacing "12,0,...,0" over 20 sections of 50),
    # i.e. the regime the guidance weights were tuned for (posterior variance ~1e-3..1e-5); every step index is <= 50, so
    # every step is guided
    dp = mk(args, gd=ref.gdp, return_class=ref.respace.SpacedDiffusionPoseNet, num_diffusion_timesteps=1000,
            timestep_respacing=POSE_RESPACING, device='cpu')
    dt = mk(args, gd=ref.gdt, return_class=ref.respace.SpacedDiffusionTrajNet, num_diffusion_timesteps=Tn_steps, device='cpu')
    dc = mk(args, gd=ref.gdt, return_class=ref.respace.SpacedDiffusionTrajNet, num_diffusion_timesteps=Tn_steps, device='cpu')
    pose, traj = synthetic.pipeline_batches(B, 71, ds_pose)
    tfd, pfd = ds_traj.traj_feat_dim, ds_traj.pose_feat_dim
    val_pose = None
    with _patched_th(ref.gdp, 72), _patched_th(ref.gdt, 73):
        for it in range(rounds):
            shape = list(traj['motion_repr_clean'][:, :, 0:tfd].shape)
            if it == 0:
                _, val_traj = dt.eval_losses(model=mt, batch=traj, shape=shape, progress=False, clip_denoised=False,
                                             timestep_respacing='', cond_fn_with_grad=True, compute_loss=False, smplx_model=body)
            else:
                traj['control_cond'] = torch.zeros([shape[0], shape[1], pfd])
                traj['control_cond'][:, 0:-1] = val_pose[:, :, 0].permute(0, 2, 1)[:, :, -pfd:]
                traj['control_cond'][:, -1] = traj['control_cond'][:, -2].clone()
                _, val_traj = dc.eval_losses(model=mc, batch=traj, shape=shape, progress=False, clip_denoised=False,
                                             timestep_respacing='', cond_fn_with_grad=True, compute_loss=False, smplx_model=body)
            comp = traj['motion_repr_clean'].clone()
            comp[..., 0], comp[..., 2:4], comp[..., 6] = val_traj[..., 0], val_traj[..., 1:3], val_traj[..., 3]
            comp[..., 7:13], comp[..., 16:19] = val_traj[..., 4:10], val_traj[..., 10:13]
            if it == 0:
                traj['motion_repr_noisy'] = comp
            full = comp.detach().numpy() * ds_traj.Std + ds_traj.Mean
            rep = _rep_dict(torch.from_numpy(full))
            joints, _ = ref.mr.recover_from_repr_smpl(rep, recover_mode='smplx_params', smplx_model=_VertsBody(body), return_verts=True)
            joints = joints.detach().numpy()
            rows = []
            for i in range(B):
                go = ref.kt.rotation_matrix_to_angle_axis(ref.quat.rot6d_to_rotmat(rep['smplx_rot_6d'][i]))
                bp = ref.kt.rotation_matrix_to_angle_axis(ref.quat.rot6d_to_rotmat(rep['smplx_body_pose_6d'][i].reshape(-1, 6)))
                d = get_repr_smplx(positions=joints[i], smplx_params_dict={
                    'transl': rep['smplx_trans'][i].numpy(), 'global_orient': go.numpy(),
                    'body_pose': bp.reshape(-1, 63).numpy(), 'betas': rep['smplx_betas'][i].numpy()}, feet_vel_thre=5e-5)
                row = np.concatenate([d[k] for k in ko.REPR_LIST], axis=-1)
                rows.append(((row - ds_pose.Mean) / ds_pose.Std)[:, 0:22])
            traj_full = torch.tensor(np.asarray(rows))
            if it == 0:
                pose['motion_repr_noisy'] = pose['motion_repr_noisy'][:, 0:-1]
                pose['motion_repr_clean'] = pose['motion_repr_clean'][:, 0:-1]
            pose['cond'] = pose['motion_repr_noisy'].clone()  # input_noise, iter2_cond_noisy_pose
            pose['cond'][:, :, 0:22] = traj_full
            ids = np.asarray([1, 2, 4, 5, 7, 8, 10, 11])      # mask_scheme 'lower', applied in every round
            for k in range(3):
                pose['cond'][:, :, 22 + ids * 3 + k] = 0.
                pose['cond'][:, :, 22 + 66 + ids * 3 + k] = 0.
            for k in range(6):
                pose['cond'][:, :, 22 + 132 + (ids - 1) * 6 + k] = 0.
            pose['cond'][:, :, -4:] = 0.
            pose['cond'] = torch.permute(pose['cond'], (0, 2, 1)).unsqueeze(-2)
            if it == 0:
                pose['motion_repr_clean'] = torch.permute(pose['motion_repr_clean'], (0, 2, 1)).unsqueeze(-2)
            # The guided chain is chaotic at this batch size (3e6-weighted gradient of a hard-masked mean over only 2 clips:
            # |x_t| reaches 1e3 and a 1e-6 perturbation grows to O(1) within three steps), so the states entering steps
            # 6, 5, 1 and 0 are recorded for teacher-forced comparison of single guided steps and of the final output.
            seen = {}
            orig = dp.p_sample_with_grad

            def recording(model, batch, x, t, **kw):
                seen[int(t[0])] = x.detach().clone()
                return orig(model, batch, x, t, **kw)

            dp.p_sample_with_grad = recording
            _, val_pose = dp.eval_losses(model=mp, batch=pose, shape=list(pose['motion_repr_clean'].shape), progress=False,
                                         clip_denoised=False, timestep_respacing='', cond_fn_with_grad=True, early_stop=False,
                                         compute_loss=False, grad_type='amass', smplx_model=body)
            dp.p_sample_with_grad = orig
            for i in POSE_RECORDED_STEPS:
                out[f"r{it}_xt{i}"] = seen[i].numpy()
            out[f"r{it}_val_traj"] = val_traj.detach().numpy()
            out[f"r{it}_traj_full"] = traj_full.numpy().astype(np.float32)
            out[f"r{it}_cond"] = pose['cond'].detach().numpy()
            out[f"r{it}_val_pose"] = val_pose.detach().numpy()
            print(f"pipeline round {it}: |val_traj| {float(val_traj.abs().max()):.3f} |val_pose| {float(val_pose.abs().max()):.3f}")
    out["meta"] = np.array([B, Tn_steps, Pn_steps, rounds, 71, 72, 73])
    np.savez_compressed(os.path.join(OUT, "pipeline.npz"), **out)
    print("pipeline.npz")


class _VertsBody(nn.Module):
    """The driver asks for vertices (return_verts=True) and discards them; hand back a placeholder of the right shape."""

    def __init__(self, inner):
        super().__init__()
        self.inner = inner

    def forward(self, **kw):
        o = self.inner(**kw)
        o.vertices = torch.zeros(o.joints.shape[0], 10475, 3)
        return o


# Short windows keep the fixture small; the per-window computation is the same at every clip_len.
WINDOW_CLIP = 24
WINDOW_LENGTHS = (47, 24, 16)
# (overlap, recordings) of each case: the video loaders' overlap 2 over all three (two windows of the first), the AMASS
# loader's 0 over the first (one window)
WINDOW_CASES = ((2, (0, 1, 2)), (0, (0,)))
# frames whose hips and shoulders coincide: no heading, so the reference repairs their root quaternion (one per window)
WINDOW_NAN_FRAMES = {0: (10, 35), 1: (23,)}


def window_recordings(seed=81):
    """Synthetic recordings for the window encoder: SMPL-X parameters, and FK joints of the synthetic body whose hips,
    shoulders and feet are then placed by hand so that every sign and threshold the encoder decides has a margin:

    * the body's heading phi(t) sets hips (1, 2) and shoulders (16, 17) around the pelvis; recording 0 starts facing
      -y (phi(0) near 180 deg) and turns by up to pi - 0.04 within a window without crossing pi, recording 1 faces near
      -180 deg;
    * the feet (7, 8, 10, 11) cycle through heights 0, 0.10, 0.165, 0.30 above a floor below every other joint, in
      segments of 4 frames, at per-frame steps of 0.003, 0.005, 0.009, 0.02: squared speeds and heights at least 38 %
      and 0.015 away from foot_detect's thresholds (5e-5; 0.18, 0.15), and the floor is a foot at height 0 in every window.
    """
    g = np.random.default_rng(seed)
    model = synthetic.smplx_like_model(0)
    params, joints = {k: [] for k in ("global_orient", "transl", "betas", "body_pose")}, []
    for r, n in enumerate(WINDOW_LENGTHS):
        t = np.arange(n, dtype=np.float64)
        if r == 0:
            phi = np.pi - 0.02 + 3.10 * (1 - np.cos(2 * np.pi * t / 44)) / 2
        elif r == 1:
            phi = -np.pi + 0.02 + 0.3 * np.sin(2 * np.pi * t / 19)
        else:
            phi = 0.5 * t / n
        tilt = 0.05 * np.sin(t / 13.0)
        rz = np.stack([np.zeros(n), np.zeros(n), phi], -1)
        rx = np.stack([tilt, np.zeros(n), np.zeros(n)], -1)
        go = (ref_rotation.from_rotvec(rz) * ref_rotation.from_rotvec(rx)).as_rotvec()
        transl = np.stack([0.8 * np.sin(t / 40.0) + r, 0.02 * t - r, 0.9 + 0.02 * np.sin(t / 7.0)], -1)
        betas = np.repeat(0.5 * g.standard_normal((1, 10)), n, axis=0)
        body_pose = 0.2 * g.standard_normal((n, 63))
        f = lambda a: torch.from_numpy(np.asarray(a, np.float32))
        j, _ = ko.smplx_forward(model, f(go), f(body_pose), f(betas), f(transl), return_verts=False)
        j = j[:, 0:22].numpy().astype(np.float64)
        right = np.stack([np.cos(phi), np.sin(phi), np.zeros(n)], -1)
        up = np.array([0.0, 0.0, 1.0])
        p0 = j[:, 0]
        j[:, 2], j[:, 1] = p0 + 0.10 * right - 0.05 * up, p0 - 0.10 * right - 0.05 * up
        j[:, 17], j[:, 16] = p0 + 0.18 * right + 0.45 * up, p0 - 0.18 * right + 0.45 * up
        for fr in WINDOW_NAN_FRAMES.get(r, ()):
            j[fr, 1], j[fr, 16] = j[fr, 2], j[fr, 17]
        floor = np.delete(j, [7, 8, 10, 11], axis=1)[..., 2].min() - 0.05
        levels, steps = (0.0, 0.10, 0.165, 0.30), (0.003, 0.005, 0.009, 0.02)
        for k, jj in enumerate((7, 10, 8, 11)):
            seg = (t.astype(int) // 4) + 2 * k
            z = floor + np.array(levels)[seg % 4]
            step = np.array(steps)[(seg // 4 + k) % 4]
            ang = 0.37 * t + k
            d = np.stack([step * np.cos(ang), step * np.sin(ang)], -1)  # frame t -> t + 1 moves by step[t]
            xy = p0[0:1, 0:2] + 0.1 * k + np.concatenate([np.zeros((1, 2)), np.cumsum(d, axis=0)[:-1]], axis=0)
            j[:, jj] = np.concatenate([xy, z[:, None]], -1)
        for k, v in (("global_orient", go), ("transl", transl), ("betas", betas), ("body_pose", body_pose)):
            params[k].append(np.asarray(v, np.float32))
        joints.append(j.astype(np.float32))
    return {k: np.concatenate(v) for k, v in params.items()}, np.concatenate(joints)


def gen_windows(ref):
    """The reference's loaders cut, canonicalise and encode each window of the synthetic recordings above
    (cano_seq_smplx -> get_repr_smplx, dataloader_amass.py:152-211); points_coord_trans with the inverse transf_matrix
    takes each window's canonical pose frames back to the world (eval_prox_egobody.py:177-182)."""
    params, joints = window_recordings()
    off = np.concatenate([[0], np.cumsum(WINDOW_LENGTHS)])
    out = {"lengths": np.array(WINDOW_LENGTHS, np.int64), "clip_len": np.array(WINDOW_CLIP), "joints": joints}
    out.update({f"param_{k}": v for k, v in params.items()})
    for c, (overlap, recs) in enumerate(WINDOW_CASES):
        table, tfs, reps, worlds = [], [], [], []
        for r in recs:
            n, k = WINDOW_LENGTHS[r], 0
            while k * (WINDOW_CLIP - overlap) + WINDOW_CLIP <= n:  # dataloader_video.py:167-172
                s = k * (WINDOW_CLIP - overlap)
                rows = slice(off[r] + s, off[r] + s + WINDOW_CLIP)
                p = {key: v[rows].copy() for key, v in params.items()}
                cano, cano_p, tf = ref.mr.cano_seq_smplx(positions=joints[rows].copy(), smplx_params_dict=p,
                                                         return_transf_mat=True)
                d = ref.mr.get_repr_smplx(positions=cano, smplx_params_dict=cano_p, feet_vel_thre=5e-5)
                rep = np.concatenate([d[key] for key in ko.REPR_LIST], axis=-1)
                assert np.isfinite(rep).all(), (r, s)
                # margins of the decisions an fp32 encoder has to reproduce
                for pair, hf in ((ref.mr.fid_l, (0.18, 0.15)), (ref.mr.fid_r, (0.18, 0.15))):
                    v2 = ((cano[1:, pair] - cano[:-1, pair]) ** 2).sum(-1)
                    assert np.abs(v2 / 5e-5 - 1).min() > 0.3, (r, s)
                    assert np.abs(cano[:-1, pair, 2] - np.array(hf)).min() > 0.01, (r, s)
                ang = rep[:, 0]
                assert np.abs(np.abs(ang) - np.pi / 2).min() > 5e-3, (r, s, np.abs(np.abs(ang) - np.pi / 2).min())
                assert np.abs(np.abs(rep[:, 1]) - np.pi).min() > 1.0, (r, s)
                table.append((r, s))
                tfs.append(tf)
                reps.append(rep.astype(np.float32))
                worlds.append(np.stack([ref.ou.points_coord_trans(cano[t], np.linalg.inv(tf)) for t in range(WINDOW_CLIP - 2)]))
                k += 1
        out[f"c{c}_meta"] = np.array([overlap] + list(recs), np.int64)
        out[f"c{c}_table"] = np.array(table, np.int64).reshape(-1, 2)
        out[f"c{c}_transf"] = np.asarray(tfs, np.float64)
        out[f"c{c}_repr"] = np.asarray(reps)
        out[f"c{c}_world"] = np.asarray(worlds).astype(np.float32)
        print(f"windows case {c}: overlap {overlap}, {len(table)} windows, |heading| up to "
              f"{float(np.abs(np.asarray(reps)[..., 0]).max()):.4f}, contacts {float(np.asarray(reps)[..., -4:].mean()):.2f}")
    out["n_cases"] = np.array(len(WINDOW_CASES))
    np.savez_compressed(os.path.join(OUT, "windows.npz"), **out)
    print("windows.npz")


# Input noise (dataloader_amass.py:156-227): 24-frame windows with overlap 2 over the first two recordings (three windows),
# each with its own noise scale relative to test_amass_full.py's level 3 (3 deg, 3 deg, 0.03 m, 0.1)
NOISE_LENGTHS = (47, 24)
NOISE_SCALES = (1.0, 1.0 / 30.0, 0.3)
NOISE_LOCK_JOINT, NOISE_NEAR_JOINT = 17, 18  # body_pose rotations (elbows: they move no foot, hip or shoulder)
NOISE_KEEP_LOCK_WINDOW = 1  # the window whose middle-angle noise on those two joints is zero


def _lock_rotvec(g, middle_deg, want):
    """A float32 rotvec whose 'zxy' middle angle is middle_deg, with random first and third angles, whose lock distance
    (float64, from the float32 values) is below 3e-8 rad (want='lock') or within 1e-5 of 1e-3 rad (want='near'): well
    clear of scipy's 1e-7 threshold either way."""
    from oracle import windows_noise_oracle as wno
    while True:
        e = [g.uniform(-170, 170), middle_deg, g.uniform(-170, 170)]
        rv = ref_rotation.from_euler('zxy', e, degrees=True).as_rotvec().astype(np.float32)
        d = float(wno.lock_distance(wno.quat_from_rotvec(rv.astype(np.float64))))
        if (want == 'lock' and d < 3e-8) or (want == 'near' and abs(d - 1e-3) < 1e-5):
            return rv


def noise_recordings(seed=91):
    """Recordings whose joints are FK of their parameters on the synthetic body, as AMASS's preprocessed joints are: the
    global orientation turns about z near +-180 deg (recording 0 from 178 deg through 180, recording 1 near -179 deg) with
    a small tilt; the translation moves slowly (0 to 4 mm per frame) so that feet come into contact; the body pose is
    smooth, except the two elbow rotations: NOISE_LOCK_JOINT is exactly at the 'zxy' gimbal lock (middle angle +90 deg on
    even frames, -90 on odd), NOISE_NEAR_JOINT 1e-3 rad from it."""
    g = np.random.default_rng(seed)
    model = synthetic.smplx_like_model(0)
    params, joints = {k: [] for k in ("global_orient", "transl", "betas", "body_pose")}, []
    near = 90.0 - np.degrees(1e-3)
    for r, n in enumerate(NOISE_LENGTHS):
        t = np.arange(n, dtype=np.float64)
        phi = (np.pi - 0.035 + 0.07 * t / n) if r == 0 else (-np.pi + 0.02 + 0.01 * np.sin(t / 5.0))
        tilt = 0.05 * np.sin(t / 13.0)
        go = (ref_rotation.from_rotvec(np.stack([0 * t, 0 * t, phi], -1)) *
              ref_rotation.from_rotvec(np.stack([tilt, 0 * t, 0 * t], -1))).as_rotvec()
        speed = 0.002 * (1 + np.sin(t / 4.0 + r))  # metres per frame, 0 .. 4 mm
        transl = np.stack([0.3 * r + np.cumsum(speed) * 0.6, np.cumsum(speed) * 0.8 - r, 0.9 + 0.002 * np.sin(t / 7.0)], -1)
        betas = np.repeat(0.5 * g.standard_normal((1, 10)), n, axis=0)
        body_pose = 0.15 * g.standard_normal((1, 63)) + 0.02 * np.sin(t[:, None] / 9.0 + np.arange(63))
        for fr in range(n):
            body_pose[fr, NOISE_LOCK_JOINT * 3:NOISE_LOCK_JOINT * 3 + 3] = _lock_rotvec(g, 90.0 if fr % 2 == 0 else -90.0, 'lock')
            body_pose[fr, NOISE_NEAR_JOINT * 3:NOISE_NEAR_JOINT * 3 + 3] = _lock_rotvec(g, near if fr % 2 else -near, 'near')
        f = lambda a: torch.from_numpy(np.asarray(a, np.float32))
        j, _ = ko.smplx_forward(model, f(go), f(body_pose), f(betas), f(transl), return_verts=False)
        for k, v in (("global_orient", go), ("transl", transl), ("betas", betas), ("body_pose", body_pose)):
            params[k].append(np.asarray(v, np.float32))
        joints.append(j[:, 0:22].numpy().astype(np.float32))
    return {k: np.concatenate(v) for k, v in params.items()}, np.concatenate(joints)


def gen_windows_noise(ref):
    """The reference's own AMASS loader with input noise (input_noise=True, sep_noise=False, load_noise=True): a
    DataloaderAMASS made with object.__new__, its clip lists set to the windows of the recordings above and its preset
    noise to the arrays below, then create_body_repr and __getitem__ for task 'pose' (repr_abs_only=False) and task
    'traj' (repr_abs_only=True).  The stub smplx body stands in for the SMPL-X model, as everywhere in this file."""
    import pickle
    import tempfile
    sys.path.insert(0, '/root/reference')
    import data_loaders.dataloader_amass as dla
    sys.path.pop(0)
    from oracle import windows_oracle as wo
    from oracle import windows_noise_oracle as wno
    params, joints = noise_recordings()
    L, overlap = WINDOW_CLIP, 2
    off = np.concatenate([[0], np.cumsum(NOISE_LENGTHS)])
    table = wo.window_table(NOISE_LENGTHS, L, overlap)
    assert len(table) == len(NOISE_SCALES), table
    g = np.random.default_rng(92)
    noise = {'transl': [], 'betas': [], 'global_orient': [], 'body_pose': []}
    for w, sc in enumerate(NOISE_SCALES):
        bp = (sc * 3.0 * g.standard_normal((L, 21, 3))).astype(np.float32)
        if w == NOISE_KEEP_LOCK_WINDOW:  # the noisy middle angle stays at the lock / 1e-3 rad from it
            bp[:, NOISE_LOCK_JOINT, 1] = 0.0
            bp[:, NOISE_NEAR_JOINT, 1] = 0.0
        else:
            # middle-angle noise of at least 2 deg: at the lock, (first, third) = (a, 0) and any other split of the same
            # rotation, e.g. (a - s, s), give noisy rotations s * |n_x| apart, so these windows pin scipy's split
            bp[:, NOISE_LOCK_JOINT, 1] = np.where(np.arange(L) % 2 == 0, 1.0, -1.0) * (2.0 + np.abs(bp[:, NOISE_LOCK_JOINT, 1]))
        noise['transl'].append((sc * 0.03 * g.standard_normal((L, 3))).astype(np.float32))
        noise['betas'].append((sc * 0.1 * g.standard_normal((L, 10))).astype(np.float32))
        noise['global_orient'].append((sc * 3.0 * g.standard_normal((L, 3))).astype(np.float32))
        noise['body_pose'].append(bp)
    noise = {k: np.asarray(v) for k, v in noise.items()}
    ds_pose = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_traj = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    d = object.__new__(dla.DataloaderAMASS)
    rows = [slice(off[r] + s, off[r] + s + L) for r, s in table]
    d.joints_clip_list = [joints[rw].copy() for rw in rows]
    d.smplx_clip_list = [np.concatenate([params['global_orient'][rw], params['transl'][rw], params['betas'][rw],
                                         params['body_pose'][rw]], axis=-1) for rw in rows]
    d.n_samples, d.spacing, d.joints_num, d.clip_len, d.device, d.split = len(rows), 1, 22, L, 'cpu', 'test'
    d.smplx_neutral = _StubBody()
    d.input_noise, d.sep_noise, d.load_noise = True, False, True
    d.loaded_smplx_noise_dict = {k: v.astype(np.float64) for k, v in noise.items()}
    d.noise_std_params_dict = {'global_orient': 3.0, 'transl': 0.03, 'body_pose': 3.0, 'betas': 0.1}
    d.repr_list_dict = {k: [] for k in ko.REPR_LIST}
    d.repr_list_dict_noisy = {k: [] for k in ko.REPR_LIST}
    d.smplx_params_list_dict = {k: [] for k in ('global_orient', 'transl', 'body_pose', 'betas')}
    d.joints_clean_list, d.joints_noisy_list = [], []
    noisy_params = []
    real_fk = d.smplx_neutral.forward

    def recording_fk(**kw):  # the noisy parameters as the FK receives them (float32)
        noisy_params.append({k: kw[k].numpy().copy() for k in ('global_orient', 'transl', 'betas', 'body_pose')})
        return real_fk(**kw)

    d.smplx_neutral.forward = recording_fk
    with tempfile.TemporaryDirectory() as tmp:
        cur = 0
        mean, std = {}, {}
        for k in ko.REPR_LIST:
            mean[k] = ds_pose.Mean[cur:cur + ko.REPR_DIM_DICT[k]]
            std[k] = ds_pose.Std[cur:cur + ko.REPR_DIM_DICT[k]]
            cur += ko.REPR_DIM_DICT[k]
        for name, v in (('AMASS_mean.pkl', mean), ('AMASS_std.pkl', std)):
            with open(os.path.join(tmp, name), 'wb') as fh:
                pickle.dump(v, fh)
        d.logdir = tmp
        d.create_body_repr()
    out = {"lengths": np.array(NOISE_LENGTHS, np.int64), "clip_len": np.array(L), "overlap": np.array(overlap),
           "joints": joints, "table": np.array(table, np.int64), "scales": np.array(NOISE_SCALES)}
    out.update({f"param_{k}": v for k, v in params.items()})
    out.update({f"noise_{k}": v for k, v in noise.items()})
    out["noisy_param_global_orient"] = np.asarray([p['global_orient'] for p in noisy_params])
    out["noisy_param_transl"] = np.asarray([p['transl'] for p in noisy_params])
    out["noisy_param_betas"] = np.asarray([p['betas'] for p in noisy_params])
    out["noisy_param_body_pose"] = np.asarray([p['body_pose'] for p in noisy_params]).reshape(len(rows), L, 63)
    out["noisy_joints"] = np.asarray(d.joints_noisy_list, np.float32)
    noisy_repr = np.asarray([np.concatenate([d.repr_list_dict_noisy[k][w] for k in ko.REPR_LIST], axis=-1)
                             for w in range(len(rows))])
    out["noisy_contacts"] = noisy_repr[..., 290:].astype(np.float32)
    for task, ds, abs_only in (('pose', ds_pose, False), ('traj', ds_traj, True)):
        d.task, d.repr_abs_only = task, abs_only
        d.traj_feat_dim, d.pose_feat_dim = ds.traj_feat_dim, ds.pose_feat_dim
        d.Mean, d.Std = ds.Mean, ds.Std
        items = [d.__getitem__(w) for w in range(len(rows))]
        # motion_repr_clean is windows.npz's business; noisy_joints is stored once above
        for key in set(items[0]) - {'motion_repr_clean', 'noisy_joints'}:
            out[f"{task}_{key}"] = np.asarray([it[key] for it in items])
        assert all(np.array_equal(it['noisy_joints'], out["noisy_joints"][w]) for w, it in enumerate(items))
    # margins of the noisy contact decisions (the noisy joints are canonical already)
    nj = out["noisy_joints"].astype(np.float64)
    feet = [7, 10, 8, 11]
    v2 = ((nj[:, 1:, feet] - nj[:, :-1, feet]) ** 2).sum(-1)
    hz = nj[:, :-1, feet, 2] - np.array([0.18, 0.15, 0.18, 0.15])
    out["noisy_speed_margin"] = np.abs(v2 / 5e-5 - 1)
    out["noisy_height_margin"] = np.abs(hz)
    lab = out["noisy_contacts"]
    np.savez_compressed(os.path.join(OUT, "windows_noise.npz"), **out)
    print(f"windows_noise.npz: {len(rows)} windows, noisy contacts {float(lab.mean()):.2f}, per window "
          f"{lab.mean(axis=(1, 2)).round(2).tolist()}, speed margin {float(out['noisy_speed_margin'].min()):.2e}, "
          f"height margin {float(out['noisy_height_margin'].min()):.2e}")


# The video loader (DataloaderVideo): 24-frame windows, overlap 2.  Each case is one recording, as the loader takes one:
# (name, dataset, scene from the reference's floor tables, view, frames, use_scene_floor_height, floor override)
VIDEO_CLIP = 24
VIDEO_Q_TRIALS = 4  # random float64 windows through the reference's cano_seq_smplx_egobody
ABS_CHANNELS = (0, 2, 3, 6, 7, 8, 9, 10, 11, 12, 16, 17, 18)  # repr_abs_only's trajectory channels
VIDEO_CASES = (("N3Office_00034_01", 'prox', 'N3Office', None, 46, True, None),
               ("Werkraum_03403_01", 'prox', 'Werkraum', None, 24, True, 0.0),    # a preset floor of 0.0: window minimum
               ("recording_20210907_S02_S01_01", 'egobody', 'seminar_g110', 'master', 24, True, None),
               ("recording_20210911_S07_S06_02", 'egobody', 'seminar_d78', 'sub_2', 46, False, None))
# PROX's colour camera (Kinect v2, k1 k2 p1 p2 k3) and EgoBody's per-view ones (k1 k2 p1 p2 k3 k4 k5 k6)
VIDEO_PROX_CAM = {'f': [1060.53, 1060.38], 'c': [951.30, 536.77],
                  'camera_mtx': [[1060.53, 0.0, 951.30], [0.0, 1060.38, 536.77], [0.0, 0.0, 1.0]],
                  'k': [0.0548, -0.0489, 0.0009, -0.0012, 0.0102]}
VIDEO_EGO_CAM = {'f': [918.72, 918.64], 'c': [956.13, 548.89],
                 'camera_mtx': [[918.72, 0.0, 956.13], [0.0, 918.64, 548.89], [0.0, 0.0, 1.0]],
                 'k': [0.4761, -2.7413, 0.0004, -0.0002, 1.5812, 0.3563, -2.5628, 1.5138]}


def _rigid(rotvec, t):
    m = np.eye(4)
    m[:3, :3] = ref_rotation.from_rotvec(rotvec).as_matrix()
    m[:3, 3] = t
    return m


def video_recording(g, n, cam2world, y_up, heading):
    """Camera-frame SMPL-X fits of a body that walks in the scene with its heading near `heading` (radians about the
    scene's up axis) and a small tilt, so that after the camera transform the global rotation is near pi; FK on the
    synthetic body gives the pelvis offset delta_T = pelvis - transl, which the scene -> camera inversion keeps."""
    model = synthetic.smplx_like_model(0)
    t = np.arange(n, dtype=np.float64)
    phi = heading + 0.03 * np.sin(t / 5.0)
    go_z = (ref_rotation.from_rotvec(np.stack([0 * t, 0 * t, phi], -1)) *
            ref_rotation.from_rotvec(np.stack([0.05 * np.sin(t / 13.0), 0 * t, 0 * t], -1)))
    T_z = np.stack([0.6 * np.sin(t / 30.0), 0.004 * t, 0.9 + 0.01 * np.sin(t / 7.0)], -1)
    betas = np.repeat(0.5 * g.standard_normal((1, 10)), n, axis=0).astype(np.float32)
    body_pose = (0.15 * g.standard_normal((1, 63)) + 0.05 * np.sin(t[:, None] / 6.0 + np.arange(63))).astype(np.float32)
    f = lambda a: torch.from_numpy(np.asarray(a, np.float32))
    j0, _ = ko.smplx_forward(model, f(np.zeros((n, 3))), f(body_pose), f(betas), f(np.zeros((n, 3))), return_verts=False)
    delta = j0[:, 0].numpy().astype(np.float64)
    Qm = np.array([[1.0, 0, 0], [0, 0, -1], [0, 1, 0]])
    go_s, T_s = go_z, T_z
    if y_up:  # the body walks in a y-up scene: Q^T of the z-up motion
        go_s = ref_rotation.from_matrix(Qm.T) * go_z
        T_s = (T_z + delta) @ Qm - delta
    Rc, tc = cam2world[:3, :3], cam2world[:3, 3]
    go_c = (ref_rotation.from_matrix(Rc.T) * go_s).as_rotvec()
    T_c = (T_s + delta - tc) @ Rc - delta
    return {'global_orient': go_c.astype(np.float32), 'transl': T_c.astype(np.float32), 'betas': betas,
            'body_pose': body_pose}


def video_keypoints(g, n, no_person=()):
    """OpenPose BODY_25 rows [n,25,3] (float32): pixels over the image, its corners and far outside it; confidences with
    0.2f and its float32 neighbours; frames in no_person have no person (zeros)."""
    xy = np.stack([g.uniform(0, 1920, (n, 25)), g.uniform(0, 1080, (n, 25))], -1)
    xy[0, 8], xy[0, 12] = (0.0, 0.0), (1919.0, 1079.0)
    xy[1, 9], xy[1, 13] = (0.0, 1079.0), (1919.0, 0.0)
    xy[2, 8], xy[2, 1] = (-6000.0, 9000.0), (12000.0, -7000.0)  # far outside: OpenCV's negative icdist branch
    conf = g.uniform(0, 1, (n, 25))
    c2 = np.float32(0.2)
    conf[:, 5] = c2
    conf[:, 2] = np.nextafter(c2, np.float32(1))
    conf[:, 6] = np.nextafter(c2, np.float32(0))
    kp = np.concatenate([xy, conf[..., None]], -1).astype(np.float32)
    for fr in no_person:
        kp[fr] = 0
    return kp


def gen_windows_video(ref):
    """The reference's own DataloaderVideo on tiny PROX and EgoBody recordings written to a temporary directory in the
    loader's layout (per-frame 000.pkl fits and keypoint jsons, mask_joint.npy, cam2world / calibration jsons, Color.json,
    egobody_rohm_info.csv and data_splits.csv, AMASS_mean / std.pkl), for task 'pose' (repr_abs_only False) and 'traj'
    (repr_abs_only True).  The stub smplx body stands in for the neutral and gendered SMPL-X models."""
    import json
    import pickle
    import tempfile
    sys.path.insert(0, '/root/reference')
    import data_loaders.dataloader_video as dlv
    sys.path.pop(0)
    g = np.random.default_rng(111)
    ds_pose = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_traj = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    assert ds_traj.traj_feat_dim == len(ABS_CHANNELS)
    out = {"clip_len": np.array(VIDEO_CLIP), "overlap": np.array(2), "n_cases": np.array(len(VIDEO_CASES))}
    for key, cam in (("prox", VIDEO_PROX_CAM), ("egobody", VIDEO_EGO_CAM)):
        out[f"{key}_f"], out[f"{key}_c"] = np.array(cam['f']), np.array(cam['c'])
        out[f"{key}_camera_mtx"], out[f"{key}_k"] = np.array(cam['camera_mtx']), np.array(cam['k'])

    def dump(path, obj, mode='w'):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, mode) as fh:
            (pickle.dump if mode == 'wb' else json.dump)(obj, fh)

    def write_fits(root, prm, n):
        for fr in range(n):
            dump(os.path.join(root, f"frame_{fr:05d}", "000.pkl"), {k: v[fr:fr + 1] for k, v in prm.items()}, 'wb')

    with tempfile.TemporaryDirectory() as tmp:
        base, init = os.path.join(tmp, "base"), os.path.join(tmp, "init")
        logs = {}
        # one set of statistics for both tasks (the pose model's): the rows are then the same and stored once
        for task, ds in (("pose", ds_pose), ("traj", ds_pose)):
            logs[task] = os.path.join(tmp, f"log_{task}")
            cur, mean, std = 0, {}, {}
            for k in ko.REPR_LIST:
                mean[k], std[k] = ds.Mean[cur:cur + ko.REPR_DIM_DICT[k]], ds.Std[cur:cur + ko.REPR_DIM_DICT[k]]
                cur += ko.REPR_DIM_DICT[k]
            dump(os.path.join(logs[task], "AMASS_mean.pkl"), mean, 'wb')
            dump(os.path.join(logs[task], "AMASS_std.pkl"), std, 'wb')
        dump(os.path.join(base, "calibration", "Color.json"), VIDEO_PROX_CAM)
        ego = [c for c in VIDEO_CASES if c[1] == 'egobody']
        import pandas as pd
        os.makedirs(base, exist_ok=True)
        pd.DataFrame({'recording_name': [c[0] for c in ego], 'target_idx': [1, 0], 'target_gender': ['male', 'female'],
                      'view': [c[3] for c in ego], 'scene_name': [c[2] for c in ego],
                      'body_idx_fpv': ['1 male', '1 male']}).to_csv(os.path.join(base, "egobody_rohm_info.csv"))
        pd.DataFrame({'train': ['a', 'b'], 'val': ['c', 'd'], 'test': [ego[0][0], ego[1][0]]}).to_csv(
            os.path.join(base, "data_splits.csv"))
        for view in ('master', 'sub_2'):
            dump(os.path.join(base, "kinect_cam_params", f"kinect_{view}", "Color.json"), VIDEO_EGO_CAM)
        saved_floor = {}
        for c, (name, dataset, scene, view, n, use_floor, floor_override) in enumerate(VIDEO_CASES):
            y_up = dataset == 'egobody'
            # cameras: PROX looks down at the room from 2.5 m; EgoBody's master and a sub view 60 deg around it
            cam = _rigid([-2.0, 0.3, 0.4], [1.0 + 0.1 * c, -2.0, 2.5]) if not y_up else \
                _rigid([0.2, 2.9, 0.1], [0.5, 1.4, 2.0 + 0.2 * c])
            master = cam
            if view not in (None, 'master'):
                sub2main = _rigid([0.05, 1.05, -0.02], [1.8, 0.02, 0.9])
                cam = master @ sub2main
            heading = (np.pi - 0.02) if c % 2 == 0 else (-np.pi + 0.015)
            prm = video_recording(g, n, cam, y_up, heading)
            no_person = (3, 17) if c in (0, 3) else ()
            kp = video_keypoints(g, n, no_person)
            mask = g.uniform(0, 1, (n, 25)) > 0.15
            mask[4, 7] = mask[5, 8] = mask[6, 10] = mask[7, 11] = False  # a zero on each foot joint
            mask[8:12, [7, 8, 10, 11]] = True
            kp[8:12, [14, 11, 19, 20, 21, 22, 23, 24], 2] = 0.9  # feet seen on frames 8-11: both contact masks occur
            if y_up:
                fit_dir = os.path.join(init, name, "body_idx_1" if c == 2 else "body_idx_0", "results")
                gt_root = os.path.join(base, "smplx_interactee_test" if c == 2 else "smplx_camera_wearer_test", name,
                                       "body_idx_1" if c == 2 else "body_idx_0", "results")
                gt = video_recording(g, n, master, True, heading + 0.1)
                write_fits(gt_root, gt, n)
                calib = os.path.join(base, "calibrations", name, "cal_trans")
                dump(os.path.join(calib, "kinect12_to_world", scene + ".json"), {'trans': master.tolist()})
                if view != 'master':
                    dump(os.path.join(calib, "kinect_13to12_color.json"), {'trans': sub2main.tolist()})
                kp_dir = os.path.join(base, "keypoints_cleaned", name, view)
                mask_path = os.path.join(base, "mask_joint", name, view, "mask_joint.npy")
            else:
                fit_dir = os.path.join(init, name, "results")
                dump(os.path.join(base, "cam2world", scene + ".json"), cam.tolist())
                kp_dir = os.path.join(base, "keypoints_openpose", name)
                mask_path = os.path.join(base, "mask_joint", name, "mask_joint.npy")
            write_fits(fit_dir, prm, n)
            body_idx = 1 if c == 2 else 0
            for fr in range(n):
                people = [] if fr in no_person else [{'pose_keypoints_2d': [0.0] * 75}] * body_idx + \
                    [{'pose_keypoints_2d': kp[fr].reshape(-1).tolist()}]
                dump(os.path.join(kp_dir, f"frame_{fr:05d}_keypoints.json"), {'people': people})
            os.makedirs(os.path.dirname(mask_path), exist_ok=True)
            np.save(mask_path, mask)
            table = dlv.prox_floor_height if dataset == 'prox' else dlv.egobody_floor_height
            if floor_override is not None:
                saved_floor[scene] = table[scene]
                table[scene] = floor_override
            items = {}
            try:
                for task in ("pose", "traj"):
                    d = dlv.DataloaderVideo(dataset=dataset, init_root=init, base_dir=base, body_model_path='',
                                            recording_name=name, use_scene_floor_height=use_floor,
                                            repr_abs_only=task == 'traj', task=task, overlap_len=2, clip_len=VIDEO_CLIP,
                                            logdir=logs[task], device='cpu')
                    items[task] = [d[w] for w in range(len(d))]
                if floor_override is not None:  # the same recording without a preset floor: the same windows
                    d0 = dlv.DataloaderVideo(dataset=dataset, init_root=init, base_dir=base, body_model_path='',
                                             recording_name=name, use_scene_floor_height=False, task='pose',
                                             overlap_len=2, clip_len=VIDEO_CLIP, logdir=logs['pose'], device='cpu')
                    for a, b in zip(items['pose'], [d0[w] for w in range(len(d0))]):
                        assert np.array_equal(a['transf_matrix'], b['transf_matrix'])
                        assert np.array_equal(a['motion_repr_noisy'], b['motion_repr_noisy'])
            finally:
                for k, v in saved_floor.items():
                    table[k] = v
                saved_floor.clear()
            fl = table[scene] if (use_floor and floor_override is None) else (floor_override or 0.0)
            out[f"c{c}_meta"] = np.array([int(y_up), n, int(view not in (None, 'master'))])
            out[f"c{c}_name"] = np.array(name)
            out[f"c{c}_floor"] = np.array(fl if use_floor else 0.0)
            out[f"c{c}_cam2world"], out[f"c{c}_master2world"] = cam, master
            out[f"c{c}_keypoints25"], out[f"c{c}_depth_mask"] = kp, mask
            out[f"c{c}_kp_float64"] = np.array(len(no_person) > 0)
            for k, v in prm.items():
                out[f"c{c}_param_{k}"] = v
            if y_up:
                for k, v in gt.items():
                    out[f"c{c}_gt_{k}"] = v
            pose, traj = items["pose"], items["traj"]
            for key in pose[0]:
                if key == 'frame_name':
                    assert [it['frame_name'][0] for it in pose] == [f"frame_{s:05d}" for s in range(0, n - VIDEO_CLIP + 1,
                                                                                                     VIDEO_CLIP - 2)]
                    continue
                if key == 'cano_smplx_params_dict':
                    for k in ('global_orient', 'transl', 'betas', 'body_pose'):
                        out[f"c{c}_cano_{k}"] = np.asarray([it[key][k] for it in pose])
                    continue
                out[f"c{c}_{key}"] = np.asarray([it[key] for it in pose])
                assert all(np.array_equal(np.asarray(a[key]), np.asarray(b[key])) for a, b in zip(pose, traj)), key
            for a in traj:  # the TrajNet inputs are channels of the same rows (repr_abs_only True)
                assert np.array_equal(a['cond'], a['motion_repr_noisy'][:, list(ABS_CHANNELS)])
                assert np.array_equal(a['control_cond'], a['motion_repr_noisy'][:, -ds_traj.pose_feat_dim:])
            print(f"windows_video case {c} ({dataset}, {name}): {len(pose)} windows, floor {fl}, "
                  f"keypoints dtype {pose[0]['keypoints_2d'].dtype}")
    # the EgoBody canonical frame as the reference computes it, in float64 on random joints and parameters (both floor
    # modes): the tests hold T_z Q and cano_seq_smplx of Q p against these (DESIGN §4.14)
    gq = np.random.default_rng(9)
    for trial in range(VIDEO_Q_TRIALS):
        j = gq.standard_normal((4, 22, 3))
        p = {"global_orient": gq.standard_normal((4, 3)), "transl": gq.standard_normal((4, 3)),
             "betas": gq.standard_normal((4, 10)), "body_pose": gq.standard_normal((4, 63))}
        floor = 0.0 if trial % 2 else float(gq.uniform(-2, -0.5))
        cano, cano_p, tf = ref.mr.cano_seq_smplx_egobody(j.copy(), {k: v.copy() for k, v in p.items()},
                                                         preset_floor_height=floor or None, return_transf_mat=True)
        out[f"q{trial}_joints"], out[f"q{trial}_floor"] = j, np.array(floor)
        out[f"q{trial}_global_orient"], out[f"q{trial}_transl"] = p['global_orient'], p['transl']
        out[f"q{trial}_cano_joints"], out[f"q{trial}_transf"] = cano, tf
        out[f"q{trial}_cano_global_orient"], out[f"q{trial}_cano_transl"] = cano_p['global_orient'], cano_p['transl']
    out["q_trials"] = np.array(VIDEO_Q_TRIALS)
    np.savez_compressed(os.path.join(OUT, "windows_video.npz"), **out)
    print("windows_video.npz", os.path.getsize(os.path.join(OUT, "windows_video.npz")), "bytes")


# The video driver in miniature: one recording per case cut into two 17-frame windows (17 + 15 frames), the shipped
# video flags (sample_iter 2, iter2_cond_noisy_traj / iter2_cond_noisy_pose False, early_stop), a 10-step TrajNet and
# the 12-step respaced PoseNet of gen_pipeline (every step guided)
VIDEO_PIPE_CASES = (("N3Office_00034_01", 'prox', 'N3Office'), ("recording_20210907_S02_S01_01", 'egobody', 'seminar_g110'))
# Short windows keep the fixture small (every stored [windows, 294, frames] state scales with the window): the driver's
# computation is the same at every window length whose trajectory frames are a multiple of 16, and the GPU tests run the
# 145-frame windows of encode_video through the same rounds.
VIDEO_PIPE_CLIP = 17
VIDEO_PIPE_FRAMES = VIDEO_PIPE_CLIP + VIDEO_PIPE_CLIP - 2
VIDEO_PIPE_RECORDED_STEPS = (1, 0)
# the batch keys the video driver reads (test_prox_egobody.py:185-354), stored per case; the trajectory batch's cond and
# control_cond are channels of its motion_repr_noisy (asserted), so only the rows are stored
VIDEO_PIPE_POSE_KEYS = ('motion_repr_noisy', 'mask_vec_vis', 'mask_joint_vis', 'keypoints_2d', 'transf_matrix',
                        'focal_length', 'camera_center', 'noisy_joints_scene_coord')
VIDEO_PIPE_TRAJ_KEYS = ('motion_repr_noisy',)


def gen_video_pipeline(ref):
    """The call sequence of test_prox_egobody.py:214-354 through the UNMODIFIED reference, on windows its own
    DataloaderVideo cut from recordings written to a temporary directory (the layout of gen_windows_video): TrajNet ->
    host glue on motion_repr_noisy -> PoseNet conditioned on the visibility-masked noisy rows with 2-D projection and
    skating guidance (grad_type 'prox') -> reconstruction, 2 rounds (round 2 through TrajControl)."""
    import json
    import pickle
    import tempfile
    sys.path.insert(0, '/root/reference')
    import data_loaders.dataloader_video as dlv
    sys.path.pop(0)
    get_repr_smplx = ref.mr.get_repr_smplx
    g = np.random.default_rng(121)
    tn_steps, rounds = 10, 2
    ds_pose = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_traj = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    body = _StubBody()
    mp, _ = build_ref_posenet(ref, seed=1)
    mp.dataset, mp.device = ds_pose, 'cpu'
    mt, _ = build_ref_trajnet(ref, seed=2, control=False)
    mc, _ = build_ref_trajnet(ref, seed=4, control=True)
    args = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    mk = ref.model_util.create_gaussian_diffusion
    dp = mk(args, gd=ref.gdp, return_class=ref.respace.SpacedDiffusionPoseNet, num_diffusion_timesteps=1000,
            timestep_respacing=POSE_RESPACING, device='cpu')
    dt = mk(args, gd=ref.gdt, return_class=ref.respace.SpacedDiffusionTrajNet, num_diffusion_timesteps=tn_steps, device='cpu')
    dc = mk(args, gd=ref.gdt, return_class=ref.respace.SpacedDiffusionTrajNet, num_diffusion_timesteps=tn_steps, device='cpu')
    n = VIDEO_PIPE_FRAMES
    out = {"meta": np.array([len(VIDEO_PIPE_CASES), tn_steps, 12, rounds, n, VIDEO_PIPE_CLIP]),
           "recorded_steps": np.array(VIDEO_PIPE_RECORDED_STEPS)}

    def dump(path, obj, mode='w'):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, mode) as fh:
            (pickle.dump if mode == 'wb' else json.dump)(obj, fh)

    def write_fits(root, prm):
        for fr in range(n):
            dump(os.path.join(root, f"frame_{fr:05d}", "000.pkl"), {k: v[fr:fr + 1] for k, v in prm.items()}, 'wb')

    with tempfile.TemporaryDirectory() as tmp:
        base, init = os.path.join(tmp, "base"), os.path.join(tmp, "init")
        logs = {}
        for task, ds in (("pose", ds_pose), ("traj", ds_traj)):
            logs[task] = os.path.join(tmp, f"log_{task}")
            cur, mean, std = 0, {}, {}
            for k in ko.REPR_LIST:
                mean[k], std[k] = ds.Mean[cur:cur + ko.REPR_DIM_DICT[k]], ds.Std[cur:cur + ko.REPR_DIM_DICT[k]]
                cur += ko.REPR_DIM_DICT[k]
            dump(os.path.join(logs[task], "AMASS_mean.pkl"), mean, 'wb')
            dump(os.path.join(logs[task], "AMASS_std.pkl"), std, 'wb')
        dump(os.path.join(base, "calibration", "Color.json"), VIDEO_PROX_CAM)
        dump(os.path.join(base, "kinect_cam_params", "kinect_master", "Color.json"), VIDEO_EGO_CAM)
        import pandas as pd
        ego = [c for c in VIDEO_PIPE_CASES if c[1] == 'egobody']
        pd.DataFrame({'recording_name': [c[0] for c in ego], 'target_idx': [0], 'target_gender': ['male'],
                      'view': ['master'], 'scene_name': [c[2] for c in ego],
                      'body_idx_fpv': ['1 male']}).to_csv(os.path.join(base, "egobody_rohm_info.csv"))
        pd.DataFrame({'train': ['a'], 'val': ['c'], 'test': [ego[0][0]]}).to_csv(os.path.join(base, "data_splits.csv"))
        for c, (name, dataset, scene) in enumerate(VIDEO_PIPE_CASES):
            y_up = dataset == 'egobody'
            cam = _rigid([0.2, 2.9, 0.1], [0.5, 1.4, 2.0]) if y_up else _rigid([-2.0, 0.3, 0.4], [1.0, -2.0, 2.5])
            heading = np.pi - 0.02 if c == 0 else -np.pi + 0.015
            prm = video_recording(g, n, cam, y_up, heading)
            kp = video_keypoints(g, n)
            mask = g.uniform(0, 1, (n, 25)) > 0.15
            if y_up:
                fit_dir = os.path.join(init, name, "body_idx_0", "results")
                write_fits(os.path.join(base, "smplx_camera_wearer_test", name, "body_idx_0", "results"),
                           video_recording(g, n, cam, True, heading + 0.1))
                dump(os.path.join(base, "calibrations", name, "cal_trans", "kinect12_to_world", scene + ".json"),
                     {'trans': cam.tolist()})
                kp_dir = os.path.join(base, "keypoints_cleaned", name, "master")
                mask_path = os.path.join(base, "mask_joint", name, "master", "mask_joint.npy")
            else:
                fit_dir = os.path.join(init, name, "results")
                dump(os.path.join(base, "cam2world", scene + ".json"), cam.tolist())
                kp_dir = os.path.join(base, "keypoints_openpose", name)
                mask_path = os.path.join(base, "mask_joint", name, "mask_joint.npy")
            write_fits(fit_dir, prm)
            for fr in range(n):
                dump(os.path.join(kp_dir, f"frame_{fr:05d}_keypoints.json"),
                     {'people': [{'pose_keypoints_2d': kp[fr].reshape(-1).tolist()}]})
            os.makedirs(os.path.dirname(mask_path), exist_ok=True)
            np.save(mask_path, mask)
            loaders = {task: dlv.DataloaderVideo(dataset=dataset, init_root=init, base_dir=base, body_model_path='',
                                                 recording_name=name, use_scene_floor_height=True,
                                                 repr_abs_only=task == 'traj', task=task, overlap_len=2,
                                                 clip_len=VIDEO_PIPE_CLIP,
                                                 logdir=logs[task], device='cpu') for task in ("pose", "traj")}
            items = {task: [d[w] for w in range(len(d))] for task, d in loaders.items()}
            assert len(items['pose']) == 2, len(items['pose'])
            stack = lambda its, key: torch.from_numpy(np.asarray([it[key] for it in its]))
            pose = {k: stack(items['pose'], k) for k in VIDEO_PIPE_POSE_KEYS + (('gt_joints_scene_coord',) if y_up else ())}
            traj = {k: stack(items['traj'], k) for k in ('motion_repr_noisy', 'cond', 'control_cond')}
            assert torch.equal(traj['cond'], traj['motion_repr_noisy'][..., list(ABS_CHANNELS)])
            assert torch.equal(traj['control_cond'], traj['motion_repr_noisy'][..., -ds_traj.pose_feat_dim:])
            for k, v in list(pose.items()) + [('traj_' + k, traj[k]) for k in VIDEO_PIPE_TRAJ_KEYS]:
                # the PROX loader's undistorted keypoints are float64, as the reference's guidance reads them: kept so
                assert k == 'keypoints_2d' or v.dtype == torch.float32, (k, v.dtype)
                out[f"c{c}_{'' if k.startswith('traj_') else 'pose_'}{k}"] = v.numpy()
            # one camera per recording: the reference's guidance reads dataset.cam_R / cam_t
            ds_pose.cam_R, ds_pose.cam_t = loaders['pose'].cam_R, loaders['pose'].cam_t
            c2w = torch.eye(4)
            c2w[:3, :3], c2w[:3, 3] = ds_pose.cam_R, ds_pose.cam_t.reshape(3)
            out[f"c{c}_cam2world"] = c2w.numpy()
            out[f"c{c}_meta"] = np.array([int(y_up), len(items['pose'])])
            B = len(items['pose'])
            tfd, pfd = ds_traj.traj_feat_dim, ds_traj.pose_feat_dim
            val_pose = None
            with _patched_th(ref.gdp, 130 + c), _patched_th(ref.gdt, 140 + c):
                for it in range(rounds):
                    shape = list(traj['motion_repr_noisy'][:, :, 0:tfd].shape)
                    if it == 0:
                        _, val_traj = dt.eval_losses(model=mt, batch=traj, shape=shape, progress=False, clip_denoised=False,
                                                     timestep_respacing='', compute_loss=False, cond_fn_with_grad=True,
                                                     smplx_model=body)
                    else:
                        traj['control_cond'] = torch.zeros([shape[0], shape[1], pfd])
                        traj['control_cond'][:, 0:-1] = val_pose[:, :, 0].permute(0, 2, 1)[:, :, -pfd:]
                        traj['control_cond'][:, -1] = traj['control_cond'][:, -2].clone()
                        _, val_traj = dc.eval_losses(model=mc, batch=traj, shape=shape, progress=False, clip_denoised=False,
                                                     timestep_respacing='', cond_fn_with_grad=True, compute_loss=False,
                                                     smplx_model=body)
                    comp = traj['motion_repr_noisy'].clone()
                    comp[..., 0], comp[..., 2:4], comp[..., 6] = val_traj[..., 0], val_traj[..., 1:3], val_traj[..., 3]
                    comp[..., 7:13], comp[..., 16:19] = val_traj[..., 4:10], val_traj[..., 10:13]
                    if it == 0:
                        traj['motion_repr_noisy'] = comp
                    if it < rounds - 1:  # iter2_cond_noisy_traj False
                        traj['cond'] = val_traj
                    full = comp.detach().numpy() * ds_traj.Std + ds_traj.Mean
                    rep = _rep_dict(torch.from_numpy(full))
                    joints, _ = ref.mr.recover_from_repr_smpl(rep, recover_mode='smplx_params', smplx_model=_VertsBody(body),
                                                             return_verts=True)
                    joints = joints.detach().numpy()
                    rows = []
                    for i in range(B):
                        go = ref.kt.rotation_matrix_to_angle_axis(ref.quat.rot6d_to_rotmat(rep['smplx_rot_6d'][i]))
                        bp = ref.kt.rotation_matrix_to_angle_axis(
                            ref.quat.rot6d_to_rotmat(rep['smplx_body_pose_6d'][i].reshape(-1, 6)))
                        d = get_repr_smplx(positions=joints[i], smplx_params_dict={
                            'transl': rep['smplx_trans'][i].numpy(), 'global_orient': go.numpy(),
                            'body_pose': bp.reshape(-1, 63).numpy(), 'betas': rep['smplx_betas'][i].numpy()},
                            feet_vel_thre=5e-5)
                        row = np.concatenate([d[k] for k in ko.REPR_LIST], axis=-1)
                        rows.append(((row - ds_pose.Mean) / ds_pose.Std)[:, 0:22])
                    traj_full = torch.tensor(np.asarray(rows))
                    if it == 0:
                        pose['motion_repr_noisy'] = pose['motion_repr_noisy'][:, 0:-1]
                        src = pose['motion_repr_noisy'].clone()
                    else:  # iter2_cond_noisy_pose False: the previous PoseNet output (a permuted view, as the driver)
                        src = val_pose[:, :, 0].permute(0, 2, 1)
                    pose['cond'] = src
                    pose['cond'][:, :, 0:22] = traj_full
                    if it < 1:  # mask_iter_num = 1
                        pose['cond'] = pose['cond'] * pose['mask_vec_vis'][:, 0:-2, :]
                        pose['cond'][:, :, -4:] = 0.
                    if it == 0:
                        pose['motion_repr_noisy'] = torch.permute(pose['motion_repr_noisy'], (0, 2, 1)).unsqueeze(-2)
                    pose['cond'] = torch.permute(pose['cond'], (0, 2, 1)).unsqueeze(-2)
                    out[f"c{c}_r{it}_cond"] = pose['cond'].detach().numpy().copy()
                    seen = {}
                    orig = dp.p_sample_with_grad

                    def recording(model, batch, x, t, **kw):
                        seen[int(t[0])] = x.detach().clone()
                        return orig(model, batch, x, t, **kw)

                    dp.p_sample_with_grad = recording
                    _, val_pose = dp.eval_losses(model=mp, batch=pose, shape=list(pose['motion_repr_noisy'].shape),
                                                 progress=False, clip_denoised=False, timestep_respacing='',
                                                 cond_fn_with_grad=True, early_stop=True, compute_loss=False,
                                                 grad_type='prox', smplx_model=body)
                    dp.p_sample_with_grad = orig
                    for i in VIDEO_PIPE_RECORDED_STEPS:
                        out[f"c{c}_r{it}_xt{i}"] = seen[i].numpy()
                    out[f"c{c}_r{it}_val_traj"] = val_traj.detach().numpy()
                    out[f"c{c}_r{it}_traj_full"] = traj_full.numpy().astype(np.float32)
                    out[f"c{c}_r{it}_val_pose"] = val_pose.detach().numpy().copy()
                    print(f"video pipeline case {c} ({dataset}) round {it}: |val_traj| {float(val_traj.abs().max()):.3f} "
                          f"|val_pose| {float(val_pose.abs().max()):.3f}")
            # :326-354: joints of the noisy input and of the reconstruction
            rec = val_pose[:, :, 0].permute(0, 2, 1).detach().numpy() * ds_pose.Std + ds_pose.Mean
            noisy = pose['motion_repr_noisy'][:, :, 0].permute(0, 2, 1).detach().numpy() * ds_pose.Std + ds_pose.Mean
            rep_n, rep_r = _rep_dict(torch.from_numpy(noisy)), _rep_dict(torch.from_numpy(rec))
            out[f"c{c}_rec_noisy"] = ref.mr.recover_from_repr_smpl(rep_n, recover_mode='smplx_params',
                                                                   smplx_model=_VertsBody(body), return_verts=True)[0].detach().numpy()
            out[f"c{c}_rec_from_abs_traj"] = ref.mr.recover_from_repr_smpl(rep_r, recover_mode='joint_abs_traj',
                                                                           smplx_model=body).detach().numpy()
            out[f"c{c}_rec_from_smpl"] = ref.mr.recover_from_repr_smpl(rep_r, recover_mode='smplx_params',
                                                                       smplx_model=_VertsBody(body),
                                                                       return_verts=True)[0].detach().numpy()
    out = {k: (v.astype(np.float32) if v.dtype == np.float64 and not k.endswith('keypoints_2d') else v)
           for k, v in out.items()}
    path = os.path.join(OUT, "video_pipeline.npz")
    np.savez_compressed(path, **out)
    print("video_pipeline.npz", os.path.getsize(path), "bytes")


# ------------------------------------------------------------------------------------------------------------ metrics
EVAL_AMASS_RUNS = (('lower', 0.0), ('full', 0.1), ('full', 0.0), ('full', 0.7))
EVAL_VIDEO_T = 20  # frames per synthetic window: the scripts take any clip length
EVAL_VIDEO_WINDOWS = (1, 2, 1, 3, 1, 1, 2, 1, 1, 1, 1, 1, 2, 1, 1, 1, 1, 1, 1)  # per recording of --recording_name all


def _eval_stubs():
    """Stand-ins for what the evaluation scripts import but do not use for their numbers: configargparse (an argparse
    shim), open3d / trimesh (empty) and pyrender (attribute lookups return a no-op class)."""
    cap = types.ModuleType('configargparse')

    class ArgParser(argparse.ArgumentParser):
        def __init__(self, config_file_parser_class=None, **kw):
            super().__init__(**kw)

        def add_argument(self, *a, is_config_file=False, **kw):
            return super().add_argument(*a, **kw)

    cap.ArgParser, cap.ArgumentDefaultsHelpFormatter, cap.YAMLConfigFileParser = \
        ArgParser, argparse.ArgumentDefaultsHelpFormatter, object
    pyrender = types.ModuleType('pyrender')
    pyrender.__getattr__ = lambda name: type(name, (), {'__init__': lambda self, *a, **k: None})
    return {'configargparse': cap, 'open3d': types.ModuleType('open3d'), 'trimesh': types.ModuleType('trimesh'),
            'pyrender': pyrender}


def _run_reference_script(name, argv):
    import runpy
    old = sys.argv
    sys.argv = [name] + argv
    sys.path.insert(0, '/root/reference')
    try:
        return runpy.run_path(os.path.join('/root/reference', name), run_name='__main__')
    finally:
        sys.argv = old
        sys.path.pop(0)


def _threshold_speed(g):
    """A float32 displacement dx with float32(|dx| * 30) == float32(0.1): a foot exactly at the speed threshold."""
    dx = np.float32(0.1 / 30)
    while np.float32(dx * np.float32(30)) != np.float32(0.1):
        dx = np.nextafter(dx, np.float32(1))
    return dx


def eval_amass_clips(g, n, T, with_nan=False):
    """Clean and reconstructed joints [n,T,22,3] with feet crossing every skating threshold, some exactly on one,
    penetrating toes, and contact labels [n,T,4] (the reconstruction's around 0.5, one exactly 0.5, one NaN)."""
    base = np.cumsum(g.normal(0, 0.004, (n, T, 1, 3)), axis=1) + g.normal(0, 0.3, (n, 1, 22, 3))
    G = base + g.normal(0, 0.002, (n, T, 22, 3))
    G[..., 2] = np.abs(G[..., 2]) + 0.2
    G[:, :, [7, 10, 8, 11], 2] = g.uniform(0.0, 0.22, (n, T, 4))
    G[:, 0, 0, 2] = 0.0  # h0 = 0 exactly, so that heights equal the joints' z
    G = G.astype(np.float32)
    P = (G + g.normal(0, 0.02, G.shape)).astype(np.float32)
    P[:, :, [10, 11], 2] = g.uniform(-0.12, 0.2, (n, T, 2))
    # exact thresholds: ankle at 0.15, toe at 0.1, a foot moving at exactly 0.1 m/s
    G[0, 10:20, 7, 2], G[0, 10:20, 10, 2] = np.float32(0.15), np.float32(0.1)
    dx = _threshold_speed(g)
    for t in range(30, min(40, T - 1), 2):
        for j in (7, 10, 8, 11):
            G[0, t, j, 0:2] = 0.0
            G[0, t + 1, j, 0:2] = (dx, 0.0)
            G[0, t, j, 2] = G[0, t + 1, j, 2] = 0.01
    P[1, 50:60] = G[1, 50:60]
    lc = (g.uniform(0, 1, (n, T, 4)) > 0.5).astype(np.float32)
    lc[0, 0, 0] = 0.5
    lr = g.uniform(0, 1, (n, T, 4)).astype(np.float32)
    lr[0, 1, 0], lr[0, 2, 1] = 0.5, np.nan
    if with_nan:
        G[0, 5, 3, 1] = np.nan  # poisons only mpjpe
        G[0, 7, 4, 2] = np.nan  # poisons h0 of clip 0
        P[1, 9, 10, 2] = np.nan
    return G, P, lc, lr


def eval_video_recordings(g, dataset, floors, T=EVAL_VIDEO_T):
    """Per recording: canonical joints [n,T,22,3], transf [n,4,4] (a rigid scene -> canonical map), and for EgoBody the
    scene ground truth [n,T+2,22,3] and visibility [n,T,22]; the scene feet hover around the recording's floor."""
    up, horiz = (1, [0, 2]) if dataset == 'egobody' else (2, [0, 1])
    out = []
    for r, n in enumerate(EVAL_VIDEO_WINDOWS):
        S = np.cumsum(g.normal(0, 0.004, (n, T + 2, 1, 3)), axis=1) + g.normal(0, 0.3, (n, 1, 22, 3))
        S = S + g.normal(0, 0.002, S.shape)
        S[..., up] = floors[r] + np.abs(S[..., up]) + 0.2
        S[:, :, [7, 10, 8, 11], up] = floors[r] + g.uniform(-0.1, 0.25, (n, T + 2, 4))
        drift = np.cumsum(g.normal(0, 0.006, (n, T + 2, 4, 2)), axis=1)
        for f, j in enumerate((7, 10, 8, 11)):
            for a, axis in enumerate(horiz):
                S[:, :, j, axis] += drift[:, :, f, a]
        transf = np.zeros((n, 4, 4))
        for w in range(n):
            transf[w, :3, :3] = ref_rotation.from_rotvec(g.normal(0, 1.0, 3)).as_matrix()
            transf[w, :3, 3] = g.normal(0, 1.0, 3)
            transf[w, 3, 3] = 1.0
        transf = transf.astype(np.float32)
        rec = np.einsum('wij,wtkj->wtki', transf[:, :3, :3].astype(np.float64), S[:, :T]) + transf[:, None, None, :3, 3]
        rec = (rec + g.normal(0, 0.01, rec.shape)).astype(np.float32)
        item = {'rec': rec, 'transf': transf}
        if dataset == 'egobody':
            item['gt'] = S.astype(np.float32)
            item['mask'] = (g.uniform(0, 1, (n, T, 22)) > 0.3).astype(np.float32)
        out.append(item)
    return out


def gen_eval_metrics(ref):
    """The unmodified eval_amass_full.py and eval_prox_egobody.py (runpy) on synthetic pickles in a temporary directory,
    with a dataset root holding egobody_rohm_info.csv, the calibration and the cam2world JSONs.  Keeps the scripts'
    per-frame arrays and final numbers, their inputs, and the floor height each recording used."""
    import json
    import pickle
    import tempfile
    sys.modules.update(_eval_stubs())
    g = np.random.default_rng(2024)
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        # ---------------------------------------------------------------- AMASS
        for tag, n, T, with_nan in (('amass', 4, 143, False), ('amass_nan', 2, 40, True)):
            G, P, lc, lr = eval_amass_clips(g, n, T, with_nan)
            out[f"{tag}_gt"], out[f"{tag}_rec"], out[f"{tag}_label_clean"], out[f"{tag}_label_rec"] = G, P, lc, lr
            repr_c, repr_r = np.zeros((n, T, 294), np.float32), np.zeros((n, T, 294), np.float32)
            repr_c[..., -4:], repr_r[..., -4:] = lc, lr
            path = os.path.join(tmp, f"{tag}.pkl")
            with open(path, 'wb') as f:
                pickle.dump({'repr_name_list': ko.REPR_LIST, 'repr_dim_dict': {}, 'rec_ric_data_clean_list': G,
                             'rec_ric_data_rec_list_from_abs_traj': P, 'rec_ric_data_rec_list_from_smpl': P,
                             'motion_repr_clean_list': repr_c, 'motion_repr_rec_list': repr_r}, f)
            runs = EVAL_AMASS_RUNS if tag == 'amass' else (('lower', 0.0),)
            for k, (scheme, ratio) in enumerate(runs):
                res = _run_reference_script('eval_amass_full.py', ['--saved_data_path', path, '--mask_scheme', scheme,
                                                                   '--traj_mask_ratio', str(ratio)])
                key = f"{tag}_run{k}"
                out[f"{key}_scheme"], out[f"{key}_ratio"] = np.array(scheme), np.float64(ratio)
                out[f"{key}_mpjpe_global"] = np.float64(np.mean(res['joints_mpjpe_global']))
                out[f"{key}_mpjpe_global_vis"] = np.float64(np.mean(res['joints_mpjpe_global_vis']))
                out[f"{key}_mpjpe_global_occ"] = np.float64(np.mean(res['joints_mpjpe_global_invis']))
                for name in ('skating_gt_ratio', 'skating_rec_ratio', 'acc_error', 'pene_freq', 'pene_dist'):
                    out[f"{key}_{name}"] = np.float64(res[name])
                out[f"{key}_contact_lbl_acc"] = np.float64(np.mean(res['contact_lbl_acc']))
                if k == 0:
                    out[f"{tag}_mpjpe"] = res['joints_mpjpe_global']
                    out[f"{tag}_contact_match"] = res['contact_lbl_acc']
                    out[f"{tag}_skating_gt"], out[f"{tag}_skating_rec"] = res['skating_gt'], res['skating_rec']
                    out[f"{tag}_accel_error"] = np.linalg.norm(res['acc_rec'] - res['acc_gt'], axis=-1)
                    out[f"{tag}_h0"] = res['min_height_gt']
                print(f"eval {tag} {scheme} {ratio}: mpjpe {out[f'{key}_mpjpe_global']:.5f} skating "
                      f"{out[f'{key}_skating_gt_ratio']:.4f}/{out[f'{key}_skating_rec_ratio']:.4f} pene "
                      f"{out[f'{key}_pene_freq']:.4f} {out[f'{key}_pene_dist']:.5f}")

        # ---------------------------------------------------------------- PROX / EgoBody
        root = os.path.join(tmp, 'dataset')
        scenes = {'prox': ['MPH1Library', 'N0Sofa', 'N3Library', 'N3Office'], 'egobody': sorted(ref.ou.egobody_floor_height)}
        for dataset in ('prox', 'egobody'):
            res_dir = os.path.join(tmp, dataset)
            os.makedirs(res_dir)
            # the recording list the script evaluates with --recording_name all, read back from the script itself
            src = open('/root/reference/eval_prox_egobody.py').read()
            names = _recording_names(src, dataset)
            rows = []
            floors = []
            for r, name in enumerate(names):
                if dataset == 'prox':
                    scene = name.split('_')[0]
                    floors.append(ref.ou.prox_floor_height[scene])
                    os.makedirs(os.path.join(root, 'cam2world'), exist_ok=True)
                    with open(os.path.join(root, 'cam2world', scene + '.json'), 'w') as f:
                        json.dump(np.eye(4).tolist(), f)
                else:
                    scene = scenes['egobody'][r % len(scenes['egobody'])]
                    floors.append(ref.ou.egobody_floor_height[scene])
                    view = 'sub_1' if r == 3 else 'master'
                    rows.append((name, 0, 100, 0, 'male', view, scene, 1))
                    cal = os.path.join(root, 'calibrations', name, 'cal_trans')
                    os.makedirs(os.path.join(cal, 'kinect12_to_world'), exist_ok=True)
                    with open(os.path.join(cal, 'kinect12_to_world', scene + '.json'), 'w') as f:
                        json.dump({'trans': np.eye(4).tolist()}, f)
                    with open(os.path.join(cal, 'kinect_11to12_color.json'), 'w') as f:
                        json.dump({'trans': np.eye(4).tolist()}, f)
            if rows:
                import pandas as pd
                pd.DataFrame(rows, columns=['recording_name', 'target_start_frame', 'target_end_frame', 'target_idx',
                                            'target_gender', 'view', 'scene_name', 'body_idx_fpv']).to_csv(
                    os.path.join(root, 'egobody_rohm_info.csv'), index=False)
            recs = eval_video_recordings(g, dataset, floors)
            for r, (name, item) in enumerate(zip(names, recs)):
                n = item['rec'].shape[0]
                save = {'repr_name_list': ko.REPR_LIST, 'repr_dim_dict': {}, 'rec_ric_data_noisy_list': item['rec'].copy(),
                        'rec_ric_data_rec_list_from_smpl': item['rec'].copy(),
                        'joints_input_scene_coord_list': item['rec'].copy(),
                        'motion_repr_rec_list': np.zeros((n, EVAL_VIDEO_T, 294), np.float32),
                        'motion_repr_noisy_list': np.zeros((n, EVAL_VIDEO_T, 294), np.float32),
                        'mask_joint_vis_list': item.get('mask', np.ones((n, EVAL_VIDEO_T, 22), np.float32)),
                        'trans_scene2cano_list': item['transf']}
                if dataset == 'egobody':
                    save['joints_gt_scene_coord_list'] = item['gt']
                    save['frame_name_list'] = np.zeros((n, EVAL_VIDEO_T), dtype='<U8')
                with open(os.path.join(res_dir, name + '.pkl'), 'wb') as f:
                    pickle.dump(save, f)
                for k, v in item.items():
                    out[f"{dataset}_r{r}_{k}"] = v
            out[f"{dataset}_floor"] = np.asarray(floors, np.float64)
            res = _run_reference_script('eval_prox_egobody.py', ['--dataset', dataset, '--dataset_root', root,
                                                                 '--saved_data_dir', res_dir, '--recording_name', 'all'])
            lists = ['skating_list', 'acc_list', 'ground_pene_freq_list', 'ground_pene_dist_list']
            if dataset == 'egobody':
                lists += ['acc_error_list', 'gmpjpe_list', 'mpjpe_list', 'mpjpe_list_vis', 'mpjpe_list_occ',
                          'joint_mask_list']
            for lst in lists:
                for r, name in enumerate(names):
                    out[f"{dataset}_r{r}_{lst}"] = res[lst][name]
            out[f"{dataset}_all_skating"] = np.float64(res['skating_list']['all'].mean())
            out[f"{dataset}_all_acc"] = np.float64(res['acc_list']['all'].mean())
            out[f"{dataset}_all_ground_pene_freq"] = np.float64(res['ground_pene_freq_list']['all'].mean())
            out[f"{dataset}_all_ground_pene_dist"] = np.float64(res['ground_pene_dist_list']['all'].mean())
            if dataset == 'egobody':
                m = res['joint_mask_list']['all']
                out["egobody_all_acc_error"] = np.float64(res['acc_error_list']['all'].mean())
                out["egobody_all_gmpjpe"] = np.float64(res['gmpjpe_list']['all'].mean())
                out["egobody_all_mpjpe"] = np.float64(res['mpjpe_list']['all'].mean())
                out["egobody_all_mpjpe_vis"] = np.float64(res['mpjpe_list_vis']['all'].sum() / m.sum())
                out["egobody_all_mpjpe_occ"] = np.float64(res['mpjpe_list_occ']['all'].sum() / (1 - m).sum())
            print(f"eval {dataset}: {len(names)} recordings, skating {out[f'{dataset}_all_skating']:.4f} acc "
                  f"{out[f'{dataset}_all_acc']:.3f}")
    path = os.path.join(OUT, "eval_metrics.npz")
    np.savez_compressed(path, **out)
    print("eval_metrics.npz", os.path.getsize(path), "bytes")


def _recording_names(src, dataset):
    """The script's --recording_name all list for `dataset`, parsed from its source (only to name the pickles)."""
    import ast
    tree = ast.parse(src)
    for node in ast.walk(tree):
        if isinstance(node, ast.If) and isinstance(node.test, ast.Compare) and \
                isinstance(node.test.comparators[0], ast.Constant) and node.test.comparators[0].value == dataset and \
                node.body and isinstance(node.body[0], ast.Assign) and \
                getattr(node.body[0].targets[0], 'id', None) == 'test_recording_name_list':
            return ast.literal_eval(node.body[0].value)
    raise RuntimeError(f"no recording list for {dataset}")


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    ref = import_reference()
    which = sys.argv[1:] or ["schedules", "posenet", "trajnet", "sampling", "kinematics", "glue", "pipeline",
                             "clip_guidance", "windows", "windows_noise", "windows_video", "video_pipeline", "eval_metrics"]
    for w in which:
        {"schedules": gen_schedules, "posenet": gen_posenet, "trajnet": gen_trajnet, "sampling": gen_sampling,
         "kinematics": gen_kinematics, "glue": gen_glue, "pipeline": gen_pipeline, "clip_guidance": gen_clip_guidance,
         "windows": gen_windows, "windows_noise": gen_windows_noise, "windows_video": gen_windows_video,
         "video_pipeline": gen_video_pipeline, "eval_metrics": gen_eval_metrics}[w](ref)
