"""Synthetic, seeded stand-ins for the assets the reference needs but that cannot ship: trained weights, AMASS
batches and the licence-gated SMPL-X model file.  Shapes and statistics follow SURVEY.md 8(d) / Appendix A / E.
Used by the tests, ``bench.py`` and ``__graft_entry__.smoke()``; everything is reproducible from an integer seed on
any machine (CPU generator), so golden fixtures only need to store seeds and outputs.
"""
from types import SimpleNamespace

import numpy as np
import torch

BODY_FEAT_DIM = 294
POSE_FEAT_DIM = 272
TRAJ_FEAT_DIM_POSE = 22   # PoseNet dataset: channels [0,22) are the trajectory block
TRAJ_FEAT_DIM_ABS = 13    # TrajNet with repr_abs_only=True

SMPLX_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 15, 15, 15,
                 20, 25, 26, 20, 28, 29, 20, 31, 32, 20, 34, 35, 20, 37, 38,
                 21, 40, 41, 21, 43, 44, 21, 46, 47, 21, 49, 50, 21, 52, 53]


def synth_state_dict(template, seed):
    """Deterministic random weights for every floating tensor of ``template`` (a state dict or a module).

    Matrices / conv kernels ~ N(0, 1/fan_in); biases ~ N(0, 0.02^2... scaled 0.1); norm gains 1 + N(0, 0.1^2); norm
    biases N(0, 0.1^2).  Zero-initialised TrajControl convolutions get real values too (otherwise the branch is a
    no-op and tests nothing).  Buffers named ``pe`` and everything under ``smplx_model.`` are left untouched.
    Tensors are generated in key order from one CPU generator, so the result depends only on (keys, shapes, seed)."""
    sd = template.state_dict() if hasattr(template, "state_dict") else template
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    out = {}
    for k, v in sd.items():
        if k.startswith("smplx_model.") or k.endswith(".pe") or not v.is_floating_point():
            out[k] = v.detach().clone()
            continue
        shape = tuple(v.shape)
        is_norm = (".norm" in k) or (".block.2." in k)
        if v.dim() >= 2:
            fan_in = int(np.prod(shape[1:]))
            t = torch.randn(shape, generator=g) / np.sqrt(fan_in)
        elif is_norm and k.endswith("weight"):
            t = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            t = 0.1 * torch.randn(shape, generator=g)
        out[k] = t.to(torch.float32)
    return out


def make_dataset(task="pose", seed=0, realistic_std=False):
    """The attributes of DataloaderAMASS that the models / guidance read (dataloader_amass.py:62-81, 256-263)."""
    rng = np.random.RandomState(seed)
    mean = np.zeros(BODY_FEAT_DIM, dtype=np.float32)
    std = np.ones(BODY_FEAT_DIM, dtype=np.float32)
    if realistic_std:
        mean = (0.1 * rng.randn(BODY_FEAT_DIM)).astype(np.float32)
        std = (0.1 + 0.9 * rng.rand(BODY_FEAT_DIM)).astype(np.float32)
        mean[-4:] = 0.0
        std[-4:] = 1.0
    traj = TRAJ_FEAT_DIM_POSE if task == "pose" else TRAJ_FEAT_DIM_ABS
    return SimpleNamespace(body_feat_dim=BODY_FEAT_DIM, pose_feat_dim=POSE_FEAT_DIM, traj_feat_dim=traj, joints_num=22,
                           Mean=mean, Std=std, task=task)


def posenet_batch(B, T, seed, device="cpu"):
    """x_T-independent inputs of one PoseNet sampling call: batch['cond'] [B,294,1,T] (z-scored features, contact
    channels in {0,1}) -- built the way test_amass_full.py:370 does (permute of a [B,T,C] tensor)."""
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    cond = torch.randn(B, T, BODY_FEAT_DIM, generator=g)
    cond[:, :, -4:] = (torch.rand(B, T, 4, generator=g) > 0.5).float()
    cond = cond.permute(0, 2, 1).unsqueeze(-2).contiguous()
    return {"cond": cond.to(device)}


def trajnet_batch(B, T, seed, control=False, device="cpu"):
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    batch = {"cond": torch.randn(B, T, TRAJ_FEAT_DIM_ABS, generator=g).to(device),
             "motion_repr_clean": torch.randn(B, T, BODY_FEAT_DIM, generator=g).to(device)}
    if control:
        batch["control_cond"] = torch.randn(B, T, POSE_FEAT_DIM, generator=g).to(device)
    return batch


def plausible_motion(B, T, seed, dataset=None):
    """A z-scored [B,294,1,T] motion-representation tensor whose SMPL-X part is a valid rotation sequence (6-D
    rotations from axis-angles ~ N(0, 0.3^2)), used to exercise the guidance / LBS path away from degenerate inputs."""
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    x = torch.randn(B, T, BODY_FEAT_DIM, generator=g)
    aa = 0.3 * torch.randn(B, T, 22, 3, generator=g)
    # smooth over time so that foot velocities are moderate
    aa = torch.cumsum(aa, dim=1) / torch.from_numpy(np.sqrt(np.arange(1, T + 1, dtype=np.float32)))[None, :, None, None]
    ang = aa.norm(dim=-1, keepdim=True).clamp_min(1e-8)
    k = aa / ang
    K = torch.zeros(B, T, 22, 3, 3)
    K[..., 0, 1], K[..., 0, 2] = -k[..., 2], k[..., 1]
    K[..., 1, 0], K[..., 1, 2] = k[..., 2], -k[..., 0]
    K[..., 2, 0], K[..., 2, 1] = -k[..., 1], k[..., 0]
    R = torch.eye(3) + torch.sin(ang)[..., None] * K + (1 - torch.cos(ang))[..., None] * (K @ K)
    rot6d = R[..., :, :2].reshape(B, T, 22, 6)  # row-major 3x2, matches rot6d_to_rotmat's reshape(-1,3,2)
    x[:, :, 7:13] = rot6d[:, :, 0]
    x[:, :, 154:280] = rot6d[:, :, 1:].reshape(B, T, 126)
    x[:, :, 16:19] = 0.3 * torch.cumsum(0.05 * torch.randn(B, T, 3, generator=g), dim=1)
    x[:, :, 280:290] = torch.randn(B, 1, 10, generator=g).expand(B, T, 10)
    x[:, :, 0] = 0.2 * torch.cumsum(0.05 * torch.randn(B, T, generator=g), dim=1)
    x[:, :, 2:4] = torch.cumsum(0.02 * torch.randn(B, T, 2, generator=g), dim=1)
    x[:, :, 6] = 0.9 + 0.02 * torch.randn(B, T, generator=g)
    x[:, :, 22:88] = 0.3 * torch.randn(B, 1, 66, generator=g) + torch.cumsum(0.01 * torch.randn(B, T, 66, generator=g), 1)
    x[:, :, -4:] = (torch.rand(B, T, 4, generator=g) > 0.4).float()
    if dataset is not None:
        x = (x - torch.from_numpy(dataset.Mean)) / torch.from_numpy(dataset.Std)
    return x.permute(0, 2, 1).unsqueeze(-2).contiguous()


def pipeline_batches(B, seed, ds_pose, frames=144, device="cpu"):
    """The two dataloader batches of test_amass_full.py:202-216 (pose task / traj task, repr_abs_only) on a synthetic
    plausible motion: z-scored clean representation, a noisy copy, the 13-channel absolute trajectory condition and the
    272-channel TrajControl condition.  Shared by tools/gen_golden.py, the GPU replay test and bench.py."""
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    clean = plausible_motion(B, frames, seed, ds_pose)[:, :, 0].permute(0, 2, 1).contiguous()  # [B, frames, 294]
    noisy = clean + 0.1 * torch.randn(clean.shape, generator=g)
    noisy[..., -4:] = clean[..., -4:]
    sel = [0, 2, 3, 6] + list(range(7, 13)) + list(range(16, 19))
    pose = {'motion_repr_clean': clean.clone().to(device), 'motion_repr_noisy': noisy.clone().to(device)}
    traj = {'motion_repr_clean': clean.clone().to(device), 'motion_repr_noisy': noisy.clone().to(device),
            'cond': noisy[..., sel].clone().to(device), 'control_cond': noisy[..., 22:].clone().to(device)}
    return pose, traj


def _rest_and_owner(g, J, V):
    # rest joints: a random tree embedding with bone lengths ~10-25 cm
    rest = torch.zeros(J, 3)
    for j in range(1, J):
        d = torch.randn(3, generator=g)
        rest[j] = rest[SMPLX_PARENTS[j]] + d / d.norm() * (0.08 + 0.15 * torch.rand(1, generator=g))
    # every vertex belongs to a primary bone and lies near it
    owner = torch.randint(0, J, (V,), generator=g)
    owner[:J] = torch.arange(J)
    return rest, owner


def smplx_like_faces(seed=0, num_faces=20908, num_verts=10475):
    """SMPL-X's triangle count [num_faces, 3] (int64) over the vertices of ``smplx_like_model(seed)``: each triangle joins
    three distinct vertices of one bone (the model orders its vertices by bone), so every surface stays local to a bone
    as a real mesh's does.  Bones get triangles in proportion to their vertex counts.  NOT the SMPL-X topology."""
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    J, V = 55, int(num_verts)
    _, owner = _rest_and_owner(g, J, V)
    counts = np.bincount(owner.numpy(), minlength=J)
    start = np.concatenate([[0], np.cumsum(counts)])
    rng = np.random.RandomState(int(seed))
    usable = np.nonzero(counts >= 3)[0]
    share = np.floor(num_faces * counts[usable] / counts[usable].sum()).astype(np.int64)
    share[:num_faces - int(share.sum())] += 1
    faces = []
    for j, n in zip(usable, share):
        for _ in range(int(n)):
            faces.append(start[j] + rng.choice(counts[j], 3, replace=False))
    return np.asarray(faces, np.int64).reshape(-1, 3)


def smplx_like_model(seed=0, num_verts=10475, dtype=torch.float32):
    """A synthetic body model with SMPL-X's exact tensor shapes, kinematic tree and sparsity pattern:
    v_template [V,3], shapedirs [V,3,20], posedirs [486, V*3], J_regressor [55,V] (sparse rows, convex weights),
    lbs_weights [V,55] (<= 4 bones per vertex, convex), parents[55].  NOT the licensed SMPL-X data."""
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    J, V = 55, int(num_verts)
    rest, owner = _rest_and_owner(g, J, V)
    v_template = rest[owner] + 0.05 * torch.randn(V, 3, generator=g)
    # skinning weights are spatially local in SMPL-X: a vertex is driven by its primary bone and that bone's
    # neighbours in the kinematic tree (parent, grand-parent, a child) -- not by arbitrary bones
    parent = torch.tensor([max(p, 0) for p in SMPLX_PARENTS])
    first_child = torch.arange(J)
    for j in range(J - 1, 0, -1):
        first_child[SMPLX_PARENTS[j]] = j
    neighbours = [None, parent, parent[parent], first_child]
    lbs = torch.zeros(V, J)
    for k in range(4):
        idx = owner if k == 0 else neighbours[k][owner]
        w = torch.rand(V, generator=g) * (1.0 if k == 0 else 0.3)
        lbs[torch.arange(V), idx] += w
    lbs = lbs / lbs.sum(dim=1, keepdim=True)
    # joint regressor: each joint is a convex combination of ~32 vertices owned by it (or random ones)
    Jreg = torch.zeros(J, V)
    for j in range(J):
        cand = torch.nonzero(owner == j).flatten()
        if cand.numel() < 8:
            cand = torch.randint(0, V, (32,), generator=g)
        pick = cand[torch.randperm(cand.numel(), generator=g)[:32]]
        w = torch.rand(pick.numel(), generator=g)
        Jreg[j, pick] = w / w.sum()
    shapedirs = 0.01 * torch.randn(V, 3, 20, generator=g)
    posedirs = 0.002 * torch.randn((J - 1) * 9, V * 3, generator=g)
    # real meshes index neighbouring vertices (same dominant bone) next to each other; reproduce that locality by
    # ordering the vertices by their primary bone (a pure relabelling applied consistently to every per-vertex array)
    perm = torch.sort(owner, stable=True).indices
    v_template, lbs, Jreg, shapedirs = v_template[perm], lbs[perm], Jreg[:, perm], shapedirs[perm]
    posedirs = posedirs.view(-1, V, 3)[:, perm].reshape(-1, V * 3)
    return {"v_template": v_template.to(dtype), "shapedirs": shapedirs.to(dtype), "posedirs": posedirs.to(dtype),
            "J_regressor": Jreg.to(dtype), "lbs_weights": lbs.to(dtype), "parents": list(SMPLX_PARENTS)}
