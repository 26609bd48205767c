"""Float64 reference of the length-masked foot-skating guidance (guide_skating_with_smpl over clips of different lengths),
built on the differentiable kinematics of kinematics_oracle."""
import torch

from .kinematics_oracle import FOOT_JOINTS, joints_from_abs_traj, joints_from_smplx, split_repr


def guide_skating_lengths(x0, mean, std, model, lengths, traj_feat_dim=22):
    """guide_skating over clips of lengths[b] real frames (the rest of the padded [B,294,1,T] batch is ignored): a
    velocity pair (t, t+1) of clip b counts only when t + 1 < lengths[b], the normalisers are the counts over the whole
    batch, and the gradient past each clip is zero.  A 0-dim zero tensor if nothing skates."""
    B, T = x0.shape[0], x0.shape[-1]
    x = x0.detach().clone()
    pad = torch.arange(T)[None, :] >= torch.as_tensor(lengths).reshape(B, 1)  # [B, T]
    x[pad[:, None, None, :].expand_as(x)] = 0  # padded values must not reach the autograd graph (0 x NaN = NaN)
    x.requires_grad_()
    full = x[:, :, 0].permute(0, 2, 1) * std + mean
    rep = split_repr(full)
    j_abs = joints_from_abs_traj(rep)
    j_smpl = joints_from_smplx(rep, model)
    pair_ok = (~pad[:, 1:]).to(full.dtype)[:, :, None]  # [B, T-1, 1]: both frames of the pair are real
    contact = (full[:, :, -4:].detach().clone() > 0.5).to(full.dtype)
    contact = contact[:, 0:-1] * pair_ok
    terms = []
    for j in (j_abs, j_smpl):
        vel = torch.norm((j[:, 1:, FOOT_JOINTS] - j[:, 0:-1, FOOT_JOINTS]) * 30, dim=-1)
        mask = (vel - 0.1).gt(0) * contact
        terms.append(((vel * mask).sum(), mask.sum()))
    (s_abs, n_abs), (s_smpl, n_smpl) = terms
    l_abs = s_abs / n_abs if n_abs != 0 else torch.zeros((), dtype=full.dtype)
    l_smpl = s_smpl / n_smpl if n_smpl != 0 else torch.zeros((), dtype=full.dtype)
    if n_abs != 0 or n_smpl != 0:
        g = torch.autograd.grad([-(l_smpl + l_abs)], [x])[0]
        g[:, 0:traj_feat_dim] = 0
        g[:, -4:] = 0
        g[pad[:, None, None, :].expand_as(g)] = 0
        return g
    return torch.zeros((), dtype=full.dtype)
