"""Both guidance VJPs (body.cu guide_backward_kernel through kernels_for(...).skating_guidance, glue.cu
projection_guidance_kernel through PoseNet.guide_2d_projection_with_smpl) at the 6-D rotations a denoiser's pred_xstart
carries, against the reference's autograd in float64 (kinematics_oracle.guide_skating, glue_oracle.guide_projection).

The body joints of the leg chains (1, 4, 7, 2, 5, 8) and a few others (3, 12, 16, 18) get, in every frame, one family of
6-D channels: exact identity, 1e-3 rad, 2 pi / 3 and pi - 1e-4 rotations about random axes, and non-orthonormal inputs
(columns scaled by 0.3 and 3, a2 with a 0.2-0.9 component along a1, near-collinear columns with kappa up to 1e3).  The
statistics are Mean 0 / Std 1, so the kernels read exactly these values.

Bound.  The kernels pull the rotation cotangent G back through Gram-Schmidt alone; the reference's round trip adds at most
1e-6 of the VJP (tests/test_kin_reference_host.py).  On plausible motion both kernels are within 2e-4 of the gradient's
scale (tests/test_gpu_body.py, test_gpu_glue.py); that error sits in G, and Gram-Schmidt's VJP multiplies G by at most
kappa_j = max((1 + |a2| / l2) / (2 l1), 1 / l2) (1 for orthonormal columns: dL/da1 has the terms G / l1 and
(s gu2 + (gu2.b1) a2) / l1 of size |a2| / (l1 l2), dL/da2 the term G / l2).  So channel c of joint j's 6-D block is held to
2e-4 kappa_j scale and every other channel to 2e-4 scale, with scale = max_c |reference_c| / kappa(c).
"""

import numpy as np
import pytest
import torch

import kin_reference as kr
from oracle import glue_oracle as go
from oracle import kinematics_oracle as ko
from rohm_b200 import synthetic
from rohm_b200.body_model import BodyModel, kernels_for
from rohm_b200.posenet import PoseNet

pytestmark = pytest.mark.gpu

JOINTS = (1, 4, 7, 2, 5, 8, 3, 12, 16, 18)
FAMILIES = ("identity", "1e-3 rad", "2pi/3", "pi - 1e-4", "columns x0.3, x3", "columns x3, x0.3", "a2 along a1 0.2-0.9",
            "near-collinear kappa<=1e3")


def _channels(j):
    return slice(154 + (j - 1) * 6, 154 + j * 6)


def _edge_motion(B, T, seed, family):
    """plausible_motion on unit statistics with the 6-D channels of JOINTS overwritten -> (x [B,294,1,T] float32,
    kappa per channel [294, T * B] float64 as [B, 294, T])."""
    ds = synthetic.make_dataset('pose')  # Mean 0 / Std 1
    x = synthetic.plausible_motion(B, T, seed, ds)[:, :, 0].permute(0, 2, 1).contiguous()  # [B, T, 294]
    rng = np.random.default_rng(seed)
    n = B * T * len(JOINTS)
    if family in ("identity", "1e-3 rad", "2pi/3", "pi - 1e-4"):
        r6 = kr.rot6d_of(kr.rotation_families(n, rng)[family])
    else:
        r6 = kr.nonorthonormal_families(n, rng)[family]
    r6 = torch.from_numpy(r6).float().view(B, T, len(JOINTS), 6)
    for k, j in enumerate(JOINTS):
        x[:, :, _channels(j)] = r6[:, :, k]
    kap = torch.ones(B, 294, T, dtype=torch.float64)
    for j in JOINTS:
        v = x[:, :, _channels(j)].double().reshape(-1, 6).numpy()
        a1, a2 = v[:, 0::2], v[:, 1::2]
        l1 = np.linalg.norm(a1, axis=1)
        b1 = a1 / l1[:, None]
        l2 = np.linalg.norm(a2 - (b1 * a2).sum(1, keepdims=True) * b1, axis=1)
        kj = np.maximum((1 + np.linalg.norm(a2, axis=1) / l2) / (2 * l1), 1 / l2)
        kap[:, _channels(j)] = torch.from_numpy(kj).view(B, T, 1).permute(0, 2, 1)
    return x.permute(0, 2, 1).unsqueeze(2).contiguous(), kap, ds


def _check(name, grad, ref, kap):
    """grad / ref [B, 294, 1, T]; kap [B, 294, T]."""
    grad, ref = grad[:, :, 0].double(), ref[:, :, 0].double()
    assert bool(torch.isfinite(grad).all())
    assert float(grad[:, :22].abs().max()) == 0.0 and float(grad[:, -4:].abs().max()) == 0.0
    scale = float((ref.abs() / kap).max())
    assert scale > 0
    ratio = float(((grad - ref).abs() / (kap * scale)).max())
    print(f"{name}: max |cuda - reference| / (kappa scale) = {ratio:.2e}")
    assert ratio < 2e-4, (name, ratio)


@pytest.fixture(scope="module")
def body(cuda_device):
    return BodyModel.create('', device=cuda_device, seed=0), synthetic.smplx_like_model(0)


@pytest.mark.parametrize("family", FAMILIES)
def test_skating_guidance_at_edge_rotations(body, cuda_device, family):
    bm, model = body
    B, T = 2, 40
    x, kap, ds = _edge_motion(B, T, 21, family)
    mean, std = torch.zeros(294), torch.ones(294)
    k = kernels_for(bm, cuda_device, B * T, with_vertices=False)
    grad, loss = k.skating_guidance(x.to(cuda_device), mean.to(cuda_device), std.to(cuda_device), want_loss=True)
    loss = loss.cpu()
    # both recovery paths skate, so neither half of the gradient can pass as zero; the counts equal the reference's
    full = x[:, :, 0].permute(0, 2, 1).double()
    rep = ko.split_repr(full)
    contact = (full[:, :, -4:] > 0.5).double()
    _, n_abs = ko.skating_loss_terms(ko.joints_from_abs_traj(rep), contact)
    _, n_smpl = ko.skating_loss_terms(ko.joints_from_smplx(rep, model), contact)
    assert float(n_abs) > 0 and float(n_smpl) > 0
    assert float(loss[1]) == float(n_abs) and float(loss[3]) == float(n_smpl)
    ref = ko.guide_skating(x.double(), mean.double(), std.double(), model)
    assert ref.dim() == 4
    _check(f"skating, {family}", grad.cpu(), ref, kap)


def _posenet(dev, ds):
    m = PoseNet(dataset=ds, body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4, device=dev,
                traj_feat_dim=22)
    m.load_state_dict({k: v.cpu() for k, v in synthetic.synth_state_dict(m, 1).items()})
    return m.to(dev).eval()


@pytest.mark.parametrize("family", FAMILIES)
def test_projection_guidance_at_edge_rotations(cuda_device, family):
    B, T = 2, 24
    x, kap, ds = _edge_motion(B, T, 22, family)
    g = torch.Generator().manual_seed(3)
    cam_R = torch.tensor([[1., 0, 0], [0, 0, 1], [0, -1, 0]])
    cam_t = torch.tensor([[0.2, -5.0, 1.0]])
    tm = torch.eye(4).repeat(B, 1, 1)
    tm[:, :3, 3] = 0.1 * torch.randn(B, 3, generator=g)
    focal, center = torch.tensor([[1000., 990.]]).repeat(B, 1), torch.tensor([[900., 500.]]).repeat(B, 1)
    kp2 = torch.cat([900 + 300 * torch.randn(B, T, 22, 1, generator=g), 500 + 200 * torch.randn(B, T, 22, 1, generator=g),
                     torch.rand(B, T, 22, 1, generator=g)], dim=-1)
    ref, _ = go.guide_projection(x.double(), torch.zeros(294, dtype=torch.float64), torch.ones(294, dtype=torch.float64),
                                 synthetic.smplx_like_model(0), tm.double(), cam_R.double(), cam_t.double(), focal.double(),
                                 center.double(), kp2.double())
    dev = cuda_device
    ds.cam_R, ds.cam_t = cam_R.to(dev), cam_t.to(dev)
    m = _posenet(dev, ds)
    batch = {'transf_matrix': tm.to(dev), 'focal_length': focal.to(dev), 'camera_center': center.to(dev),
             'keypoints_2d': kp2.to(dev)}
    grad = m.guide_2d_projection_with_smpl(batch, {'pred_xstart': x.to(dev)}, None, compute_grad='x_0').cpu()
    _check(f"projection, {family}", grad, ref, kap)
