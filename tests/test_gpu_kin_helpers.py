"""The rotation and trajectory helpers of rohm_b200/csrc/kin.cuh and repr.cuh, one element per thread through the kernel
probe, against float64 references (tests/kin_reference.py) evaluated on the exact float32 inputs the kernel received.

Every bound is C u s with u = 2^-24 and s the helper's conditioning at that input; the constants C are in BOUNDS and the
test prints the largest observed ratio err / (u s) of each family.  The probe compiles the helpers with the product's
flags, but each is __forceinline__, so its copy may contract FMAs differently from a product kernel: the tests hold the
helpers to float64, not to the product's bits.

  rot6d_to_mat    b1 = a1 / l1 rounds a few times: column 0 within C u.  u2 = a2 - (b1.a2) b1 loses what cancels, so
                  b2 and b3 are within C u kappa, kappa = |a2| / l2.  l1 within C u l1, l2 within C u kappa l2, s within
                  C u |a2|.
  rot6d_backward  gu2 carries b2's error times |G| / l2: dL/da2 within C u kappa |G| / l2.  dL/da1 adds s gu2 and
                  (gu2.b1) a2, of size kappa |G| / l2 each, divided by l1: within C u kappa^2 |G| / l1 + C u |G| / l1.
                  At the 1e-12 clamps (a1 = 0 or shorter than 1e-12, a2 exactly parallel to a1 or zero) the
                  reference's gradient is of size 1 / 1e-12 and the bound is C u times the row's largest entry.
  mat_to_aa       kornia's quaternion sums three entries and takes one square root per branch; the angle is an atan2 of
                  well-scaled arguments and k = 2 theta / s is relative: the vector within C u |aa| (|aa| = 0 exactly at
                  the identity).  Near pi the reference may return -aa for the same rotation (qw's sign), so there the
                  vector is compared modulo sign, and the rotation it represents within C u.
  rodrigues       sin / cos of the angle: within C u (1 + |r|) per entry (an angle of 50 carries 50 u of rounding into
                  sin and cos).  NaN exactly where the reference's is.
  rotvec_to_mat   scipy's quaternion route: within C u (1 + |r|) per entry, either side of the 1e-3 Taylor switch.
  heading_quat    across = (j1 - j2) + (j17 - j16) rounds at u |j| (|j| = the four joints' summed norms), so the
                  horizontal heading is off by u kappa_h, kappa_h = |j| / |across_xy|.  q3 within C u kappa_h; q0 = w / n
                  with w = |f| + f_y cancelling as forward nears -y, within C u (kappa_h + 1 / |q0|).
  qrot_z          within C u |v|.
  traj_channels   the angles within C u; the root velocity within C u |r1 - r0|, the angular velocity within
                  C u max|R1 - R0|, the translation velocity within C u |tr1 - tr0|; the copied channels exactly.
  clip_of_frame   exact.
"""
import math

import numpy as np
import pytest
import torch

import kernel_probe as kp
import kin_reference as kr
from rohm_b200 import glue

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("cuda_device")]

U = kr.U
# the constants C of the module docstring, per helper: 2 to 6 times the largest ratio observed on an H100 (SXM, 700 W);
# each test prints its maxima
BOUNDS = {"rot6d col0": 8, "rot6d col12": 16, "rot6d norms": 16, "rot6d backward": 16, "mat_to_aa": 8,
          "mat_to_aa rotation": 16, "round trip": 16, "rodrigues": 4, "rotvec": 4, "heading": 4, "qrot_z": 8, "traj": 8,
          "product aa": 16}


def _ratio(name, err, scale):
    """Largest err / (u scale) (rows with scale 0 must have err 0), printed and held to BOUNDS[name]."""
    err, scale = np.asarray(err, dtype=np.float64), np.asarray(scale, dtype=np.float64)
    assert np.all(np.isfinite(err)), name
    zero = scale == 0
    assert np.all(err[zero] == 0), name
    r = float((err[~zero] / (U * scale[~zero])).max()) if (~zero).any() else 0.0
    print(f"{name}: max ratio {r:.2f} (bound {BOUNDS[name]})")
    assert r <= BOUNDS[name], (name, r)
    return r


def _dev(x):
    return torch.as_tensor(np.asarray(x), dtype=torch.float32).cuda()


def _f64(t):
    return t.double().cpu().numpy()


# ------------------------------------------------------------------------------------------------------------
# rot6d_to_mat / rot6d_backward
# ------------------------------------------------------------------------------------------------------------
def _rot6d_inputs():
    """{family: float32-exact float64 [n, 6]}, plus the degenerate rows (the 1e-12 clamps) separately."""
    rng = np.random.default_rng(1)
    fam = {}
    n = 256
    a1, a2 = rng.standard_normal((n, 3)), rng.standard_normal((n, 3))
    norms = 10.0 ** rng.uniform(-6, 6, (n, 2))
    x = np.empty((n, 6))
    x[:, 0::2], x[:, 1::2] = kr.unit(a1) * norms[:, :1], kr.unit(a2) * norms[:, 1:]
    fam["norms 1e-6..1e6"] = x
    for ang in (1e-1, 1e-2, 1e-3, 1e-4, 1e-5, 1e-6):
        b1, p = kr.unit(rng.standard_normal((64, 3))), rng.standard_normal((64, 3))
        p = kr.unit(p - (p * b1).sum(1, keepdims=True) * b1)
        x = np.empty((64, 6))
        x[:, 0::2], x[:, 1::2] = b1, math.cos(ang) * b1 + math.sin(ang) * p
        fam[f"a2 at {ang:g} rad"] = x
    for name, R in kr.rotation_families(64, rng).items():
        fam[name] = kr.rot6d_of(R)
    fam.update(kr.nonorthonormal_families(64, rng))
    fam = {k: kr.f32(v).numpy() for k, v in fam.items()}
    deg = np.zeros((8, 6))
    deg[0, 1::2] = [0.3, -1.2, 0.5]                            # a1 = 0
    deg[1, 0::2] = [0.6, 0.0, -0.8]                            # a2 = 0
    deg[2, 0::2], deg[2, 1::2] = [0.0, 4.0, 0.0], [0.0, -0.5, 0.0]  # a2 = -a1 / 8, exact in float32
    deg[3, 0::2], deg[3, 1::2] = [2.0, 0.0, 0.0], [8.0, 0.0, 0.0]
    deg[4, 0::2], deg[4, 1::2] = [0.0, 0.0, -1.0], [0.0, 0.0, 0.25]
    deg[5] = 0.0                                               # both zero
    deg[6, 0::2] = [3e-13, 0.0, 0.0]                           # |a1| below the clamp
    deg[6, 1::2] = [0.0, 1.0, 0.0]
    deg[7, 0::2], deg[7, 1::2] = [1.0, 0.0, 0.0], [1.0, 3e-13, 0.0]  # l2 below the clamp
    return fam, kr.f32(deg).numpy()


ROT6D, DEGENERATE = _rot6d_inputs()


def test_rot6d_to_mat_against_float64():
    for name, x in list(ROT6D.items()) + [("degenerate", DEGENERATE)]:
        R, lls = kp.rot6d_to_mat(_dev(x))
        R, lls = _f64(R), _f64(lls)
        Rr, llr = kr.rot6d_to_mat(torch.from_numpy(x))
        Rr, llr = Rr.numpy(), llr.numpy()
        a2n = np.linalg.norm(x[:, 1::2], axis=1)
        kap = np.ones(len(x)) if name == "degenerate" else kr.kappa(x)
        print(f"[{name}]")
        _ratio("rot6d col0", np.abs(R[:, :, 0] - Rr[:, :, 0]).max(1), np.ones(len(x)))
        _ratio("rot6d col12", np.abs(R[:, :, 1:] - Rr[:, :, 1:]).max((1, 2)), kap)
        _ratio("rot6d norms", np.abs(lls[:, 0] - llr[:, 0]), llr[:, 0])
        _ratio("rot6d norms", np.abs(lls[:, 1] - llr[:, 1]), kap * llr[:, 1])
        _ratio("rot6d norms", np.abs(lls[:, 2] - llr[:, 2]), a2n)
    # the clamps: zero columns stay exactly zero, like the reference's
    R, _ = kp.rot6d_to_mat(_dev(DEGENERATE))
    Rr, _ = kr.rot6d_to_mat(torch.from_numpy(DEGENERATE))
    assert torch.equal(R.cpu() == 0, Rr.float() == 0)


def test_rot6d_backward_at_the_clamps():
    """a1 = 0, a2 = 0, a2 exactly parallel to a1, and 0 < |a1|, l2 < 1e-12: the reference divides by the clamp 1e-12, whose
    gradient is I / 1e-12 without the projection onto b's normal plane; the VJP is finite and equals it."""
    G = kr.f32(np.random.default_rng(9).standard_normal((len(DEGENERATE), 3, 3))).numpy()
    gx = _f64(kp.rot6d_backward(_dev(DEGENERATE), _dev(G)))
    ref = kr.rot6d_vjp(torch.from_numpy(DEGENERATE), torch.from_numpy(G)).numpy()
    assert np.all(np.isfinite(gx)) and np.abs(ref).max() > 1e11
    _ratio("rot6d backward", np.abs(gx - ref).max(1), np.abs(ref).max(1))


def test_rot6d_backward_against_float64_autograd():
    rng = np.random.default_rng(2)
    for name, x in ROT6D.items():
        G = kr.f32(rng.standard_normal((len(x), 3, 3))).numpy()
        gx = _f64(kp.rot6d_backward(_dev(x), _dev(G)))
        ref = kr.rot6d_vjp(torch.from_numpy(x), torch.from_numpy(G)).numpy()
        assert np.all(np.isfinite(gx)), name
        print(f"[{name}]")
        gmax = np.abs(G).max((1, 2))
        _, lls = kr.rot6d_to_mat(torch.from_numpy(x))
        l1, l2 = lls[:, 0].numpy(), lls[:, 1].numpy()
        kap = kr.kappa(x)
        _ratio("rot6d backward", np.abs(gx[:, 1::2] - ref[:, 1::2]).max(1), kap * gmax / l2)
        _ratio("rot6d backward", np.abs(gx[:, 0::2] - ref[:, 0::2]).max(1), (kap * kap + 1) * gmax / l1)


def test_round_trip_against_float64():
    """rodrigues(mat_to_aa(rot6d_to_mat(x))), the forward rotation of both guidance kernels: within C u kappa of the
    reference's round trip."""
    for name, x in ROT6D.items():
        R = _f64(kp.rot6d_round_trip(_dev(x)))
        ref = kr.round_trip(torch.from_numpy(x)).numpy()
        print(f"[{name}]")
        _ratio("round trip", np.abs(R - ref).max((1, 2)), kr.kappa(x))


# ------------------------------------------------------------------------------------------------------------
# mat_to_aa
# ------------------------------------------------------------------------------------------------------------
def _aa_inputs():
    rng = np.random.default_rng(3)
    fam = {}
    n = 64
    for th in (0.0, 1e-7, 1e-4, 2e-3 * (1 - 1e-3), 2e-3, 2e-3 * (1 + 1e-3), 0.5, 2 * math.pi / 3 - 1e-5,
               2 * math.pi / 3, 2 * math.pi / 3 + 1e-5, math.pi - 1e-2, math.pi - 1e-3, math.pi - 1e-4, math.pi - 1e-5,
               math.pi - 1e-6, math.pi):
        fam[f"angle {th:.9g}"] = kr.axis_angle_mat(kr.random_axes(n, rng), np.full(n, th))
    fam["random"] = kr.axis_angle_mat(kr.random_axes(256, rng), rng.uniform(0, math.pi, 256))
    # axes with two equal components give two equal diagonal entries: the Shepperd branches' ties
    ties = kr.unit(np.array([[1.0, 1.0, 0.3], [0.2, 1.0, 1.0], [1.0, 0.4, 1.0], [1.0, 1.0, 1.0], [1.0, -1.0, 0.0],
                             [0.0, 1.0, 1.0], [1.0, 0.0, -1.0], [1.0, 1.0, 2.0]]))
    for th in (1.0, 2 * math.pi / 3, 2.5, math.pi - 1e-4, math.pi):
        fam[f"tied diagonal {th:.6g}"] = kr.axis_angle_mat(ties, np.full(len(ties), th))
    # pi exactly about each axis and about diagonal axes: R = 2 n n^T - I, exactly symmetric
    axes = kr.unit(np.array([[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0], [1.0, 1.0, 0], [0, 1.0, 1.0], [1.0, 0, 1.0],
                             [1.0, 1.0, 1.0], [1.0, -1.0, 1.0], [-1.0, 1.0, 1.0]]))
    fam["pi about axes"] = 2 * axes[:, :, None] * axes[:, None, :] - np.eye(3)[None]
    return {k: kr.f32(v).numpy() for k, v in fam.items()}


AA = _aa_inputs()


def test_mat_to_aa_against_float64():
    for name, R in AA.items():
        aa = _f64(kp.mat_to_aa(_dev(R)))
        ref = kr.mat_to_aa(torch.from_numpy(R)).numpy()
        norm = np.linalg.norm(ref, axis=1)
        err = np.abs(aa - ref).max(1)
        near_pi = norm > 3.0
        err[near_pi] = np.minimum(err, np.abs(aa + ref).max(1))[near_pi]  # -aa is the same rotation at pi
        print(f"[{name}]")
        _ratio("mat_to_aa", err, norm)
        rot = kr.rodrigues(torch.from_numpy(aa)).numpy()
        rot_ref = kr.rodrigues(torch.from_numpy(ref)).numpy()
        _ratio("mat_to_aa rotation", np.abs(rot - rot_ref).max((1, 2)), np.ones(len(R)))


def test_mat_to_aa_takes_every_branch():
    """The families reach the trace > 0 branch and all three diagonal branches, and both signs of qw near pi."""
    R = np.concatenate(list(AA.values()))
    tr = R[:, 0, 0] + R[:, 1, 1] + R[:, 2, 2]
    b1 = (tr <= 0) & (R[:, 0, 0] > R[:, 1, 1]) & (R[:, 0, 0] > R[:, 2, 2])
    b2 = (tr <= 0) & ~b1 & (R[:, 1, 1] > R[:, 2, 2])
    b3 = (tr <= 0) & ~b1 & ~b2
    assert (tr > 0).any() and b1.any() and b2.any() and b3.any()
    ref = kr.mat_to_aa(torch.from_numpy(R)).numpy()
    assert (np.linalg.norm(ref, axis=1) > math.pi - 1e-5).any()


def test_product_rot6d_to_angle_axis_agrees_with_the_probe():
    """glue.rot6d_to_angle_axis (the product's rot6d_to_aa_kernel) and the probe's mat_to_aa(rot6d_to_mat(x)) hold the
    same bound against float64 on every 6-D edge input."""
    rows = [x for x in ROT6D.values()] + [kr.f32(kr.rot6d_of(R)).numpy() for R in AA.values()]
    x = np.concatenate(rows)
    ref = kr.mat_to_aa(kr.rot6d_to_mat(torch.from_numpy(x))[0]).numpy()
    norm = np.linalg.norm(ref, axis=1)
    kap = kr.kappa(x)
    Rp, _ = kp.rot6d_to_mat(_dev(x))
    probe = _f64(kp.mat_to_aa(Rp))
    prod, Rprod = glue.rot6d_to_angle_axis(_dev(x), want_rotmat=True)
    prod = _f64(prod)
    for name, aa in (("probe", probe), ("product", prod)):
        err = np.abs(aa - ref).max(1)
        near_pi = norm > 3.0
        err[near_pi] = np.minimum(err, np.abs(aa + ref).max(1))[near_pi]
        print(f"[{name}]")
        # the Gram-Schmidt rounding (u kappa) moves the rotation the vector is read from
        _ratio("product aa", err, kap * np.maximum(norm, 1.0))


# ------------------------------------------------------------------------------------------------------------
# rodrigues / rotvec_to_mat
# ------------------------------------------------------------------------------------------------------------
def _rotvecs(rng, mags):
    return np.concatenate([kr.random_axes(32, rng) * m for m in mags])


def test_rodrigues_against_float64():
    rng = np.random.default_rng(4)
    r = _rotvecs(rng, (0.0, 1e-9, 1e-6, 1e-3, 1.0, math.pi, 2 * math.pi, 50.0))
    # components near -1e-8, where r + 1e-8 cancels: exactly -1e-8 in all three (the zero vector, NaN), in some, and a
    # few float32 ulps away
    e = np.float32(1e-8)
    near = []
    for k in range(-3, 4):
        v = np.float32(e)
        for _ in range(abs(k)):
            v = np.nextafter(v, np.float32(np.inf) if k > 0 else np.float32(0))
        near.append([-v, -e, -e])
        near.append([-v, -v, -v])
    near += [[-e, -e, 0.0], [-e, 0.0, 0.0], [-e, -e, 1e-3], [-e, -e, -e]]
    r = kr.f32(np.concatenate([r, np.asarray(near, dtype=np.float64)])).numpy()
    R = _f64(kp.rodrigues(_dev(r)))
    ref = kr.rodrigues(torch.from_numpy(r)).numpy()
    nan, nan_ref = np.isnan(R).any((1, 2)), np.isnan(ref).any((1, 2))
    assert np.array_equal(nan, nan_ref) and nan_ref.sum() >= 2
    assert np.array_equal(np.isnan(R), np.isnan(ref))
    ok = ~nan_ref
    _ratio("rodrigues", np.abs(R[ok] - ref[ok]).max((1, 2)), 1.0 + np.linalg.norm(r[ok], axis=1))


def test_rotvec_to_mat_against_float64():
    rng = np.random.default_rng(5)
    a = np.float32(1e-3)
    mags = [a]
    lo, hi = a, a
    for _ in range(4):
        lo, hi = np.nextafter(lo, np.float32(0)), np.nextafter(hi, np.float32(1))
        mags += [lo, hi]
    r = [np.eye(3)[k % 3] * float(m) for k, m in enumerate(mags)]  # |r| is the float32 value itself
    r = np.concatenate([np.asarray(r), _rotvecs(rng, [float(m) for m in mags] + [0.0, math.pi, 2 * math.pi, 1e3]),
                        rng.standard_normal((128, 3))])
    r = kr.f32(r).numpy()
    R = _f64(kp.rotvec_to_mat(_dev(r)))
    ref = kr.rotvec_to_mat(r).numpy()
    _ratio("rotvec", np.abs(R - ref).max((1, 2)), 1.0 + np.linalg.norm(r, axis=1))


# ------------------------------------------------------------------------------------------------------------
# heading_quat / qrot_z / traj_channels
# ------------------------------------------------------------------------------------------------------------
def _heading_joints(across, rng):
    """Four float32 joints at about 1 m whose across vector is `across` (before the joints' rounding)."""
    n = len(across)
    p, q = rng.uniform(-1, 1, (n, 3)), rng.uniform(-1, 1, (n, 3))
    j = [p + across / 2, p, q + across / 2, q]  # (j1 - j2) + (j17 - j16) = across
    return [kr.f32(v).numpy() for v in j]


def test_heading_quat_against_float64():
    rng = np.random.default_rng(6)
    across = []
    for h in (1.0, 1e-1, 1e-2, 1e-3, 1e-4, 1e-5, 1e-6):  # horizontal part of a unit across vector
        phi = rng.uniform(-math.pi, math.pi, 32)
        across.append(np.stack([h * np.cos(phi), h * np.sin(phi), np.full(32, math.sqrt(1 - h * h))], 1))
    # forward within 1e-4 rad of -y: across_xy = -(cos d, sin d)
    d = np.concatenate([10.0 ** rng.uniform(-6, -4, 16), -(10.0 ** rng.uniform(-6, -4, 16))])
    across.append(np.stack([-np.cos(d), -np.sin(d), rng.uniform(-0.5, 0.5, 32)], 1))
    across = np.concatenate(across)
    j1, j2, j17, j16 = _heading_joints(across, rng)
    # exactly vertical across (no horizontal part) and forward exactly -y (across along -x): NaN, as in the reference's
    nan_rows = np.array([[[0.3, -0.2, 1.0], [0.3, -0.2, 0.0], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]],
                         [[0.3, -0.2, 1.0], [0.3, -0.2, 0.5], [-1.0, 2.0, 0.1], [-1.0, 2.0, 0.7]],
                         [[-1.0, 0.0, 0.4], [0.0, 0.0, 0.0], [0.25, 0.0, -1.0], [0.25, 0.0, 0.0]],
                         [[-0.5, 0.0, 0.0], [0.0, 0.0, 0.0], [-0.5, 0.0, 0.0], [0.0, 0.0, 0.0]]])
    nan_rows = kr.f32(nan_rows).numpy()
    j1, j2, j17, j16 = (np.concatenate([t, nan_rows[:, k]]) for k, t in enumerate((j1, j2, j17, j16)))
    q = _f64(kp.heading_quat(*(_dev(t) for t in (j1, j2, j17, j16))))
    ref = kr.heading_quat(j1, j2, j17, j16)
    nan_ref = np.isnan(ref).any(1)
    assert np.array_equal(np.isnan(q), np.isnan(ref)) and nan_ref.sum() == 4
    ok = ~nan_ref
    acr = (j1 - j2) + (j17 - j16)
    jsum = sum(np.linalg.norm(t, axis=1) for t in (j1, j2, j17, j16))
    kap_h = (jsum / np.linalg.norm(acr[:, :2], axis=1))[ok]
    q, ref = q[ok], ref[ok]
    assert np.all(q[:, 1] == 0)
    _ratio("heading", np.abs(q[:, 2] - ref[:, 2]), kap_h)
    _ratio("heading", np.abs(q[:, 0] - ref[:, 0]), kap_h + 1 / np.abs(ref[:, 0]))


def test_qrot_z_against_float64():
    rng = np.random.default_rng(7)
    phi = rng.uniform(-math.pi, math.pi, 256)
    wz = kr.f32(np.stack([np.cos(phi / 2), np.sin(phi / 2)], 1)).numpy()
    v = kr.f32(rng.standard_normal((256, 3)) * 10.0 ** rng.uniform(-3, 3, (256, 1))).numpy()
    out = _f64(kp.qrot_z(_dev(wz), _dev(v)))
    _ratio("qrot_z", np.abs(out - kr.qrot_z(wz, v)).max(1), np.linalg.norm(v, axis=1))


def _traj_inputs(rng):
    n = 64
    fam = {}

    def heading_q(phi):  # qbetween's quaternion (q0 >= 0) of heading phi in (-pi, pi]
        return np.stack([np.cos(phi / 2), np.sin(phi / 2)], 1)

    def pairs(phi0, phi1, R0, R1, r0, r1, t0, t1):
        return (kr.f32(np.concatenate([heading_q(phi0), heading_q(phi1)], 1)).numpy(),
                kr.f32(np.stack([r0, r1], 1)).numpy(), kr.f32(np.stack([R0, R1], 1)).numpy(),
                kr.f32(np.stack([t0, t1], 1)).numpy())

    phi0 = rng.uniform(-math.pi, math.pi, n)
    ax = kr.random_axes(n, rng)
    R0 = kr.axis_angle_mat(ax, rng.uniform(0, 3, n))
    R1 = kr.axis_angle_mat(ax, rng.uniform(0, 3, n))
    r0 = rng.standard_normal((n, 3))
    t0 = rng.standard_normal((n, 3))
    fam["generic"] = pairs(phi0, phi0 + 0.05 * rng.standard_normal(n), R0, R1, r0, r0 + 0.02 * rng.standard_normal((n, 3)),
                           t0, t0 + 0.02 * rng.standard_normal((n, 3)))
    # heading crossing +-pi between the frames (q0 of qbetween changes sign): both directions
    dlt = 10.0 ** rng.uniform(-6, -1, (n, 2))
    sgn = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    fam["heading crossing pi"] = pairs(sgn * (math.pi - dlt[:, 0]), -sgn * (math.pi - dlt[:, 1]), R0, R1, r0,
                                       r0 + 0.02 * rng.standard_normal((n, 3)), t0, t0)
    # global orientation near pi
    Rp0 = kr.axis_angle_mat(ax, np.full(n, math.pi - 1e-4))
    Rp1 = kr.axis_angle_mat(ax, np.full(n, math.pi)) @ kr.axis_angle_mat(kr.random_axes(n, rng), np.full(n, 1e-3))
    fam["orientation near pi"] = pairs(phi0, phi0, Rp0, Rp1, r0, r0, t0, t0)
    # translations of 1e3 m
    big = 1e3 * kr.unit(rng.standard_normal((n, 3)))
    fam["translation 1e3 m"] = pairs(phi0, phi0 + 1e-3, R0, R0, big, big + 0.01 * rng.standard_normal((n, 3)), big,
                                     big + 0.01 * rng.standard_normal((n, 3)))
    return fam


def test_traj_channels_against_float64():
    rng = np.random.default_rng(8)
    for name, (q, roots, rots, trs) in _traj_inputs(rng).items():
        out = _f64(kp.traj_channels(_dev(q), _dev(roots), _dev(rots), _dev(trs)))
        ref = kr.traj_channels(q, roots, rots, trs)
        print(f"[{name}]")
        exact = [2, 3, 6] + list(range(7, 13)) + [16, 17, 18]
        assert np.array_equal(out[:, exact], ref[:, exact]), name
        ones = np.ones(len(q))
        # no wrap-around: the angles match without reduction modulo 2 pi
        _ratio("traj", np.abs(out[:, 0:2] - ref[:, 0:2]).max(1), ones)
        _ratio("traj", np.abs(out[:, 4:6] - ref[:, 4:6]).max(1), np.linalg.norm(roots[:, 1] - roots[:, 0], axis=1))
        _ratio("traj", np.abs(out[:, 13:16] - ref[:, 13:16]).max(1), np.abs(rots[:, 1] - rots[:, 0]).max((1, 2)))
        _ratio("traj", np.abs(out[:, 19:22] - ref[:, 19:22]).max(1), np.linalg.norm(trs[:, 1] - trs[:, 0], axis=1))
        if name == "heading crossing pi":
            # the channel is the angle of q[t+1] q[t]^-1 as the reference forms it, without flipping q to w >= 0: across
            # the crossing qbetween's w changes sign, so the channel is -+pi plus half the small heading step, next to
            # atan2's cut, and the kernel has to land on the reference's side of it (checked above, no reduction)
            assert np.all(np.abs(ref[:, 1]) > 3.0)


# ------------------------------------------------------------------------------------------------------------
# clip_of_frame
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 2, 3, 64, 65535, 1 << 22])
def test_clip_of_frame_is_searchsorted(B):
    """Every packed frame of B clips of 1 to 5 frames (the entry points take lengths >= 1), against numpy's
    searchsorted.  B = 2^22 clips exceed every caller's frame capacity."""
    rng = np.random.default_rng(B)
    lengths = rng.integers(1, 6, B)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    frames = np.arange(off[-1], dtype=np.int32)
    got = kp.clip_of_frame(torch.from_numpy(off).cuda(), torch.from_numpy(frames).cuda()).cpu().numpy()
    want = np.searchsorted(off, frames, side="right") - 1
    assert np.array_equal(got, want)
