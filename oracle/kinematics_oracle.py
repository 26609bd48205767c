"""Oracle (test infrastructure only): rotation conversions, motion-representation recovery, SMPL-X forward and the
foot-skating guidance gradient, restated with differentiable torch-CPU ops (any float dtype).

References (sanweiliti/RoHM @ 57ba22c):
  rot6d_to_rotmat                       data_loaders/common/quaternion.py:482-501
  qinv / qrot                           data_loaders/common/quaternion.py:14-18, 52-71
  rotation_matrix_to_angle_axis chain   utils/konia_transform.py:317-340, 344-347, 350-444, 45-48, 561-631
  recover_root_rot_pos / recover_from_repr_smpl   data_loaders/motion_representation.py:285-329, 332-398
  guide_skating_with_smpl               model/posenet.py:196-257
  REPR_LIST / REPR_DIM_DICT             utils/other_utils.py:17-37
SMPL-X body model: third-party smplx==0.1.28 (environment.yml:198), NOT in the reference tree and not installable
here -> restated from the published algorithm (lbs.py: blend_shapes, vertices2joints, batch_rodrigues,
transform_mat, batch_rigid_transform, lbs; body_models.py: SMPLX.forward) as summarised in SURVEY.md Appendix E.
PARITY UNPINNED for that part (no reference tests or fixtures exist for it).
"""
import torch
import torch.nn.functional as F

REPR_LIST = ['root_rot_angle', 'root_rot_angle_vel', 'root_l_pos', 'root_l_vel', 'root_height',
             'smplx_rot_6d', 'smplx_rot_vel', 'smplx_trans', 'smplx_trans_vel',
             'local_positions', 'local_vel', 'smplx_body_pose_6d', 'smplx_betas', 'foot_contact']
REPR_DIM_DICT = {'root_rot_angle': 1, 'root_rot_angle_vel': 1, 'root_l_pos': 2, 'root_l_vel': 2, 'root_height': 1,
                 'smplx_rot_6d': 6, 'smplx_rot_vel': 3, 'smplx_trans': 3, 'smplx_trans_vel': 3,
                 'local_positions': 66, 'local_vel': 66, 'smplx_body_pose_6d': 126, 'smplx_betas': 10,
                 'foot_contact': 4}

SMPLX_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 15, 15, 15,
                 20, 25, 26, 20, 28, 29, 20, 31, 32, 20, 34, 35, 20, 37, 38,
                 21, 40, 41, 21, 43, 44, 21, 46, 47, 21, 49, 50, 21, 52, 53]


def split_repr(full):
    """[..., 294] -> dict by REPR_LIST (posenet.py:209-215)."""
    out, cur = {}, 0
    for name in REPR_LIST:
        out[name] = full[..., cur:cur + REPR_DIM_DICT[name]]
        cur += REPR_DIM_DICT[name]
    return out


# ------------------------------------------------------------------------------------------------------------
# rotations
# ------------------------------------------------------------------------------------------------------------
def rot6d_to_rotmat(x):
    x = x.reshape(-1, 3, 2)
    a1, a2 = x[:, :, 0], x[:, :, 1]
    b1 = F.normalize(a1)  # eps 1e-12
    b2 = F.normalize(a2 - torch.einsum('bi,bi->b', b1, a2).unsqueeze(-1) * b1)
    b3 = torch.cross(b1, b2, dim=1)
    return torch.stack((b1, b2, b3), dim=-1)


def _safe_div(num, den, eps=1e-6):
    den = den.clone()
    den[den.abs() < eps] += eps
    return num / den


def _safe_atan2(y, x, eps=1e-6):
    y = y.clone()
    y[(y.abs() < eps) & (x.abs() < eps)] += eps
    return torch.atan2(y, x)


def rotmat_to_quat(R, eps=1e-6):
    """konia_transform.py:350-444 (WXYZ)."""
    v = R.reshape(*R.shape[:-2], 9)
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = torch.chunk(v, 9, dim=-1)
    trace = m00 + m11 + m22

    def pos():
        sq = torch.sqrt((trace + 1.0).clamp_min(eps)) * 2.0
        return torch.cat((0.25 * sq, _safe_div(m21 - m12, sq), _safe_div(m02 - m20, sq), _safe_div(m10 - m01, sq)), -1)

    def c1():
        sq = torch.sqrt((1.0 + m00 - m11 - m22).clamp_min(eps)) * 2.0
        return torch.cat((_safe_div(m21 - m12, sq), 0.25 * sq, _safe_div(m01 + m10, sq), _safe_div(m02 + m20, sq)), -1)

    def c2():
        sq = torch.sqrt((1.0 + m11 - m00 - m22).clamp_min(eps)) * 2.0
        return torch.cat((_safe_div(m02 - m20, sq), _safe_div(m01 + m10, sq), 0.25 * sq, _safe_div(m12 + m21, sq)), -1)

    def c3():
        sq = torch.sqrt((1.0 + m22 - m00 - m11).clamp_min(eps)) * 2.0
        return torch.cat((_safe_div(m10 - m01, sq), _safe_div(m02 + m20, sq), _safe_div(m12 + m21, sq), 0.25 * sq), -1)

    w2 = torch.where(m11 > m22, c2(), c3())
    w1 = torch.where((m00 > m11) & (m00 > m22), c1(), w2)
    return torch.where(trace > 0.0, pos(), w1)


def quat_to_aa(q, eps=1e-6):
    """konia_transform.py:561-631 (WXYZ)."""
    cos_t, q1, q2, q3 = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    s2 = q1 * q1 + q2 * q2 + q3 * q3
    s = torch.sqrt(s2.clamp_min(eps))
    two_theta = 2.0 * torch.where(cos_t < 0.0, _safe_atan2(-s, -cos_t), _safe_atan2(s, cos_t))
    k = torch.where(s2 > 0.0, _safe_div(two_theta, s, eps), 2.0 * torch.ones_like(s))
    return torch.stack((q1 * k, q2 * k, q3 * k), dim=-1)


def rotmat_to_aa(R):
    return quat_to_aa(rotmat_to_quat(R))


def qinv(q):
    mask = torch.ones_like(q)
    mask[..., 1:] = -mask[..., 1:]
    return q * mask


def qrot(q, v):
    shape = list(v.shape)
    q = q.contiguous().view(-1, 4)
    v = v.contiguous().view(-1, 3)
    qvec = q[:, 1:]
    uv = torch.cross(qvec, v, dim=1)
    uuv = torch.cross(qvec, uv, dim=1)
    return (v + 2 * (q[:, :1] * uv + uuv)).view(shape)


# ------------------------------------------------------------------------------------------------------------
# SMPL-X (restated from smplx==0.1.28; see module docstring)
# ------------------------------------------------------------------------------------------------------------
def batch_rodrigues(aa):
    """lbs.py batch_rodrigues: eps is added to the VECTOR before the norm."""
    n = aa.shape[0]
    angle = torch.norm(aa + 1e-8, dim=1, keepdim=True)
    d = aa / angle
    cos, sin = torch.cos(angle)[:, None], torch.sin(angle)[:, None]
    rx, ry, rz = torch.split(d, 1, dim=1)
    zeros = torch.zeros((n, 1), dtype=aa.dtype, device=aa.device)
    K = torch.cat([zeros, -rz, ry, rz, zeros, -rx, -ry, rx, zeros], dim=1).view(n, 3, 3)
    ident = torch.eye(3, dtype=aa.dtype, device=aa.device).unsqueeze(0)
    return ident + sin * K + (1 - cos) * torch.bmm(K, K)


def batch_rigid_transform(rot_mats, joints, parents):
    """lbs.py batch_rigid_transform.  rot_mats [N,J,3,3], joints [N,J,3]."""
    N, J = joints.shape[:2]
    joints = joints.unsqueeze(-1)
    rel = joints.clone()
    rel[:, 1:] = rel[:, 1:] - joints[:, parents[1:]]
    T = torch.cat([F.pad(rot_mats.reshape(-1, 3, 3), [0, 0, 0, 1]),
                   F.pad(rel.reshape(-1, 3, 1), [0, 0, 0, 1], value=1.0)], dim=2).reshape(N, J, 4, 4)
    chain = [T[:, 0]]
    for i in range(1, J):
        chain.append(torch.matmul(chain[parents[i]], T[:, i]))
    G = torch.stack(chain, dim=1)
    posed = G[:, :, :3, 3]
    jh = F.pad(joints, [0, 0, 0, 1])
    A = G - F.pad(torch.matmul(G, jh), [3, 0, 0, 0, 0, 0, 0, 0])
    return posed, A


def smplx_forward(model, global_orient, body_pose, betas, transl, return_verts=True, dtype=None):
    """SMPLX.forward as RoHM calls it (motion_representation.py:379-389): jaw/eyes/hands/expression are zeros.
    model: dict with v_template [V,3], shapedirs [V,3,20], posedirs [486, V*3], J_regressor [55,V],
    lbs_weights [V,55], parents (list of 55).  Returns (joints [N,55,3], vertices [N,V,3] or None).
    Runs on the device of ``global_orient``; the model's tensors are moved there."""
    dtype = dtype or global_orient.dtype
    dev = global_orient.device
    m = {k: (v.to(device=dev, dtype=dtype) if torch.is_tensor(v) else v) for k, v in model.items()}
    N = global_orient.shape[0]
    full_pose = torch.cat([global_orient.reshape(N, 1, 3).to(dtype), body_pose.reshape(N, 21, 3).to(dtype),
                           torch.zeros(N, 33, 3, dtype=dtype, device=dev)], dim=1)
    shape_comps = torch.cat([betas.to(dtype), torch.zeros(N, 10, dtype=dtype, device=dev)], dim=-1)
    v_shaped = m["v_template"] + torch.einsum('bl,mkl->bmk', shape_comps, m["shapedirs"])
    J = torch.einsum('bik,ji->bjk', v_shaped, m["J_regressor"])
    R = batch_rodrigues(full_pose.reshape(-1, 3)).view(N, 55, 3, 3)
    posed, A = batch_rigid_transform(R, J, m["parents"])
    joints = posed + transl.to(dtype).unsqueeze(1)
    if not return_verts:
        return joints, None
    ident = torch.eye(3, dtype=dtype, device=dev)
    pose_feature = (R[:, 1:] - ident).reshape(N, -1)
    v_posed = v_shaped + torch.matmul(pose_feature, m["posedirs"]).view(N, -1, 3)
    Tm = torch.matmul(m["lbs_weights"], A.reshape(N, 55, 16)).view(N, -1, 4, 4)
    vh = torch.cat([v_posed, torch.ones(N, v_posed.shape[1], 1, dtype=dtype, device=dev)], dim=2)
    verts = torch.matmul(Tm, vh.unsqueeze(-1))[:, :, :3, 0]
    return joints, verts + transl.to(dtype).unsqueeze(1)


# ------------------------------------------------------------------------------------------------------------
# motion representation recovery (motion_representation.py:285-398)
# ------------------------------------------------------------------------------------------------------------
def joints_from_abs_traj(rep):
    """recover_from_repr_smpl(recover_mode='joint_abs_traj'), up_axis='z'.  rep: dict of [B,T,d]. -> [B,T,22,3]"""
    ang = rep['root_rot_angle'][..., 0]
    q = torch.zeros(ang.shape + (4,), dtype=ang.dtype)
    q[..., 0] = torch.cos(ang)
    q[..., 3] = torch.sin(ang)
    r_pos = torch.zeros(ang.shape + (3,), dtype=ang.dtype)
    r_pos[..., [0, 1]] = rep['root_l_pos']
    r_pos[..., 2] = rep['root_height'][..., 0]
    pos = rep['local_positions'][..., 3:]
    pos = pos.reshape(pos.shape[:-1] + (21, 3))
    pos = qrot(qinv(q[..., None, :]).expand(pos.shape[:-1] + (4,)), pos)
    pos = torch.cat([pos[..., 0:1] + r_pos[..., None, 0:1], pos[..., 1:2] + r_pos[..., None, 1:2], pos[..., 2:3]], dim=-1)
    return torch.cat([r_pos.unsqueeze(-2), pos], dim=-2)


def smplx_params_from_repr(rep):
    """The parameter dict of motion_representation.py:375-382."""
    go = rotmat_to_aa(rot6d_to_rotmat(rep['smplx_rot_6d'].reshape(-1, 6)))
    bp = rotmat_to_aa(rot6d_to_rotmat(rep['smplx_body_pose_6d'].reshape(-1, 6))).reshape(-1, 63)
    return {'global_orient': go, 'body_pose': bp, 'betas': rep['smplx_betas'].reshape(-1, 10),
            'transl': rep['smplx_trans'].reshape(-1, 3)}


def joints_from_smplx(rep, model, return_verts=False):
    """recover_from_repr_smpl(recover_mode='smplx_params').  -> [B,T,22,3] (and vertices [B,T,V,3])."""
    bs = rep['smplx_rot_6d'].shape[0]
    p = smplx_params_from_repr(rep)
    joints, verts = smplx_forward(model, p['global_orient'], p['body_pose'], p['betas'], p['transl'], return_verts)
    joints = joints[:, 0:22].reshape(bs, -1, 22, 3)
    if return_verts:
        return joints, verts.reshape(bs, joints.shape[1], -1, 3)
    return joints


# ------------------------------------------------------------------------------------------------------------
# guidance (posenet.py:196-257)
# ------------------------------------------------------------------------------------------------------------
FOOT_JOINTS = [7, 10, 8, 11]


def skating_loss_terms(joints, contact, fps=30, thres=0.1):
    vel = (joints[:, 1:, FOOT_JOINTS] - joints[:, 0:-1, FOOT_JOINTS]) * fps
    vel = torch.norm(vel, dim=-1)
    mask = (vel - thres).gt(0) * contact[:, 0:-1]
    return (vel * mask).sum(), mask.sum()


def guide_skating(x0, mean, std, model, traj_feat_dim=22):
    """grad of -(loss_smpl + loss_abs) w.r.t. the normalised x0 [B,294,1,T]; a 0-dim zero tensor if nothing skates."""
    x = x0.detach().clone().requires_grad_()
    full = x[:, :, 0].permute(0, 2, 1) * std + mean
    rep = split_repr(full)
    j_abs = joints_from_abs_traj(rep)
    j_smpl = joints_from_smplx(rep, model)
    contact = full[:, :, -4:].detach().clone()
    contact = (contact > 0.5).to(full.dtype)
    s_abs, n_abs = skating_loss_terms(j_abs, contact)
    s_smpl, n_smpl = skating_loss_terms(j_smpl, contact)
    l_abs = s_abs / n_abs if n_abs != 0 else torch.zeros((), dtype=full.dtype)
    l_smpl = s_smpl / n_smpl if n_smpl != 0 else torch.zeros((), dtype=full.dtype)
    if n_abs != 0 or n_smpl != 0:
        g = torch.autograd.grad([-(l_smpl + l_abs)], [x])[0]
        g[:, 0:traj_feat_dim] = 0
        g[:, -4:] = 0
        return g
    return torch.zeros((), dtype=full.dtype)
