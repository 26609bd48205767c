"""Host-only checks of the float64 helper references (tests/kin_reference.py) and of the assumption both guidance kernels
rely on.

1. The references reproduce the reference's own float32 results in tests/golden/kinematics.npz: rotmat_out within
   8 u kappa per entry (u = 2^-24, kappa = |a2| / l2 of the row: the float32 Gram-Schmidt's rounding, which the second
   and third columns amplify by kappa; observed 1.9), aa_out within 16 u |aa| per component (kornia's quaternion route
   rounds relative to the vector, near pi included; observed 2.2 from the golden matrices, 4.6 from the float64 ones).
2. Both guidance kernels (body.cu guide_backward_kernel, glue.cu projection_guidance_kernel) pull the rotation cotangent
   back through Gram-Schmidt alone, where the reference runs autograd through 6-D -> R -> axis-angle -> R.  The round trip
   is the identity on SO(3), Gram-Schmidt's output lies on SO(3), so the two VJPs agree unless one of the reference's
   clamps or offsets changes the round trip itself.  In float64 the difference, relative to the VJP's largest entry, is
     - 2e-13 at most with rodrigues' 1e-8 offset taken out and angles above the 2e-3 rad clamp (observed 4.5e-14, on
       the near-collinear kappa = 1e3 family: float64 rounding amplified by kappa);
     - 4e-8 at most with the offset (observed 1.5e-8): batch_rodrigues normalises r by |r + 1e-8 (1, 1, 1)|, so its
       output is a rotation by an angle off by up to sqrt(3) 1e-8, and the VJP moves by that much relative;
     - 1e-6 at most below the clamp, 2 sin(theta / 2) < 2e-3 (observed 4.5e-7): kornia replaces |q_vec| by
       sqrt(max(|q_vec|^2, 1e-6)) = 1e-3, which scales the vector by 1 - (1e-3)^2 / 3 + O(theta^2) and drops the
       (2/3) |q_vec|^2 <= 6.7e-7 relative derivative of k = 2 atan2(s, w) / s.
   All three are below float32 resolution of a kernel's gradient (about 8 ulps at worst), so the shortcut keeps the
   reference's semantics; the tests pin each bound per family so a change to either side shows.
"""
import math

import numpy as np
import pytest
import torch

import kin_reference as kr
from helpers import golden
from oracle import kinematics_oracle as ko


def test_references_reproduce_the_golden_rotation_chain():
    g = golden("kinematics.npz")
    r6 = torch.from_numpy(g["rot6d_in"])
    R, _ = kr.rot6d_to_mat(r6)
    kap = torch.from_numpy(kr.kappa(r6.double().numpy()))
    err = (R - torch.from_numpy(g["rotmat_out"]).double()).abs().amax(dim=(1, 2))
    ratio = err / (kr.U * kap)
    print(f"rotmat_out: max ratio to u kappa = {float(ratio.max()):.2f}")
    assert float(ratio.max()) <= 8
    aa_ref = torch.from_numpy(g["aa_out"]).double()
    scale = aa_ref.norm(dim=1)
    for name, src in (("golden", torch.from_numpy(g["rotmat_out"]).double()), ("float64", R)):
        err = (kr.mat_to_aa(src) - aa_ref).abs().amax(dim=1)
        assert bool((err[scale == 0] == 0).all())
        ratio = err[scale > 0] / (kr.U * scale[scale > 0])
        print(f"aa_out from the {name} matrices: max ratio to u |aa| = {float(ratio.max()):.2f}")
        assert float(ratio.max()) <= 16


def _vjp_pair(x, G, eps):
    """(round-trip VJP with rodrigues offset eps, Gram-Schmidt VJP), float64."""
    xr = x.clone().requires_grad_()
    R = kr.rodrigues(ko.rotmat_to_aa(ko.rot6d_to_rotmat(xr)), eps)
    rt = torch.autograd.grad((R * G).sum(), xr)[0]
    return rt, kr.rot6d_vjp(x, G)


def _families():
    """Every edge family of the helper and guidance tests: {name: (float64 6-D [n, 6], smallest rotation angle)}."""
    rng = np.random.default_rng(11)
    n = 64
    out = {}
    angles = {"identity": 0.0, "1e-3 rad": 1e-3, "2pi/3": 2 * math.pi / 3, "pi - 1e-4": math.pi - 1e-4}
    for name, R in kr.rotation_families(n, rng).items():
        out[name] = (kr.rot6d_of(R), angles[name])
    for name, x in kr.nonorthonormal_families(n, rng).items():
        out[name] = (x, 0.1)  # rotation angles drawn from [0.1, 3]
    for th in (1e-7, 1e-4, 2e-3 * (1 - 1e-3), 2e-3 * (1 + 1e-3), 2 * math.pi / 3 + 1e-5, 2 * math.pi / 3 - 1e-5,
               math.pi - 1e-2, math.pi - 1e-6, math.pi):
        out[f"angle {th:.9g}"] = (kr.rot6d_of(kr.axis_angle_mat(kr.random_axes(n, rng), np.full(n, th))), th)
    # axes that make two diagonal entries equal (the Shepperd branches' ties), near and at pi
    ties = kr.unit(np.array([[1.0, 1.0, 0.3], [0.2, 1.0, 1.0], [1.0, 0.4, 1.0], [1.0, 1.0, 1.0]]))
    for th in (2.5, math.pi - 1e-4, math.pi):
        out[f"tied diagonal {th:.6g}"] = (kr.rot6d_of(kr.axis_angle_mat(ties, np.full(len(ties), th))), th)
    return out


FAMILIES = _families()


@pytest.mark.parametrize("name", list(FAMILIES))
def test_round_trip_vjp_equals_the_gram_schmidt_vjp(name):
    x, theta = FAMILIES[name]
    x = torch.from_numpy(x)
    G = torch.from_numpy(np.random.default_rng(5).standard_normal((x.shape[0], 3, 3)))
    rt, gs = _vjp_pair(x, G, kr.EPS_RODRIGUES)
    scale = float(gs.abs().max())
    assert scale > 0 and bool(torch.isfinite(rt).all())
    err = float((rt - gs).abs().max()) / scale
    clamped = 2 * math.sin(theta / 2) < 2e-3
    print(f"{name}: |round trip - Gram-Schmidt| / scale = {err:.3e}")
    assert err <= (1e-6 if clamped else 4e-8)
    if theta > 0 and not clamped:
        rt0, _ = _vjp_pair(x, G, 0.0)
        err0 = float((rt0 - gs).abs().max()) / scale
        print(f"{name}: without the rodrigues offset = {err0:.3e}")
        assert err0 <= 2e-13
