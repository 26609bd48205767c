"""Float64 reference of the guidance with per-clip normalisers (PoseNet.guidance_normaliser = 'clip'): each clip of a padded
[B,294,1,T] batch goes through the existing restatements alone, as a one-clip batch of its own n_b frames (n_b = lengths[b],
or T without lengths).  Frames past a clip are never read and get a zero gradient."""
import torch

from . import glue_oracle, masked_skating_oracle


def _clip_lengths(x0, lengths):
    B, T = x0.shape[0], x0.shape[-1]
    return [T] * B if lengths is None else [int(v) for v in lengths]


def guide_skating_per_clip(x0, mean, std, model, lengths=None, traj_feat_dim=22):
    """Clip b's skating gradient is guide_skating on x0[b:b+1, ..., :n_b] alone (masked_skating_oracle with one clip of
    n_b frames, i.e. the unmasked reference on that clip); zero where nothing of the clip skates and past the clip."""
    g = torch.zeros(x0.shape, dtype=x0.dtype)
    for b, n in enumerate(_clip_lengths(x0, lengths)):
        gb = masked_skating_oracle.guide_skating_lengths(x0[b:b + 1, ..., :n], mean, std, model, [n], traj_feat_dim)
        if gb.dim() > 0:
            g[b:b + 1, ..., :n] = gb
    return g


def guide_projection_per_clip(x0, mean, std, model, transf_matrix, cam_R, cam_t, focal, center, keypoints_2d, lengths=None,
                              traj_feat_dim=22):
    """Clip b's 2-D projection gradient and loss are glue_oracle.guide_projection on clip b alone (its n_b frames, its
    transf_matrix / focal / center row and its first n_b keypoint frames) -> (grad [B,294,1,T], loss [B])."""
    g = torch.zeros(x0.shape, dtype=x0.dtype)
    losses = []
    for b, n in enumerate(_clip_lengths(x0, lengths)):
        gb, lb = glue_oracle.guide_projection(x0[b:b + 1, ..., :n], mean, std, model, transf_matrix[b:b + 1], cam_R, cam_t,
                                              focal[b:b + 1], center[b:b + 1], keypoints_2d[b:b + 1, :n], traj_feat_dim)
        g[b:b + 1, ..., :n] = gb
        losses.append(lb)
    return g, torch.stack(losses)
