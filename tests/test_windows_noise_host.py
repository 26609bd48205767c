"""CPU: the float64 oracle of the windows' input noise (oracle/windows_oracle.py encode_noisy) against the reference's own
AMASS loader with preset noise, pinned by tests/golden/windows_noise.npz (tools/gen_golden.py gen_windows_noise); the
oracle's 'zxy' Euler extraction against scipy at, near and away from the gimbal lock; and the refusals of
windows.InputNoise and of the noisy encode that need no device."""
import warnings

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from helpers import golden
from oracle import windows_noise_oracle as wno
from oracle import windows_oracle as wo
from rohm_b200 import synthetic, windows
from rohm_b200._lib import RohmB200Error

PARAM_NAMES = ("global_orient", "transl", "betas", "body_pose")
LOCK_JOINT, NEAR_JOINT = 17, 18  # tools/gen_golden.py NOISE_LOCK_JOINT / NOISE_NEAR_JOINT
KEEP_LOCK_WINDOW = 1  # tools/gen_golden.py NOISE_KEEP_LOCK_WINDOW


def noise_case(g):
    """(clip_len, overlap, lengths, params, joints, noise) of windows_noise.npz."""
    params = {k: g[f"param_{k}"] for k in PARAM_NAMES}
    noise = {k: g[f"noise_{k}"] for k in PARAM_NAMES}
    return int(g["clip_len"]), int(g["overlap"]), [int(n) for n in g["lengths"]], params, g["joints"], noise


def zscored_items(g, rep_noisy, rep_clean, ds_pose, ds_traj):
    """DataloaderAMASS.__getitem__ (dataloader_amass.py:317-341) on un-normalised rows: {name: array} as the fixture
    stores them."""
    pose = rep_noisy.copy()
    pose[..., 0:ds_pose.traj_feat_dim] = rep_clean[..., 0:ds_pose.traj_feat_dim]
    zp = (pose - ds_pose.Mean) / ds_pose.Std
    zt = (rep_noisy - ds_traj.Mean) / ds_traj.Std
    zc = (rep_clean - ds_traj.Mean) / ds_traj.Std
    return {"pose_motion_repr_noisy": zp, "traj_motion_repr_noisy": zt,
            "traj_cond": zt[..., list(windows.ABS_TRAJ_CHANNELS)], "traj_control_cond": zc[..., -ds_traj.pose_feat_dim:]}


def test_oracle_matches_reference_noisy_windows():
    g = golden("windows_noise.npz")
    L, overlap, lengths, params, joints, noise = noise_case(g)
    model = synthetic.smplx_like_model(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        nparams, njoints, rep = wno.encode_noisy(params, joints, lengths, noise, model, L, overlap)
    table, _, clean = wo.encode(params, joints, lengths, L, overlap)
    assert [tuple(t) for t in g["table"]] == table
    # the reference hands the FK float32 parameters; the oracle keeps float64
    for k in PARAM_NAMES:
        ref = g[f"noisy_param_{k}"].astype(np.float64)
        assert np.abs(nparams[k] - ref).max() <= 1e-6 * (1 + np.abs(ref).max()), k
    # the reference's FK runs in float32 on those float32 parameters
    assert np.abs(njoints - g["noisy_joints"]).max() < 2e-5
    ds_pose = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_traj = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    want = zscored_items(g, rep, clean, ds_pose, ds_traj)
    for name, got in want.items():
        ref = g[name].astype(np.float64)
        std = {"pose": ds_pose.Std, "traj": ds_traj.Std}[name[:4]]
        if name == "traj_cond":
            std = std[list(windows.ABS_TRAJ_CHANNELS)]
        elif name == "traj_control_cond":
            std = std[-ds_traj.pose_feat_dim:]
        # compared de-normalised, where the float32 reference carries ~1e-6 of each value
        err = np.abs(got - ref) * std / (1.0 + np.abs(ref * std))
        assert err.max() < 1e-4, (name, np.unravel_index(err.argmax(), err.shape))
    # contact labels: the oracle's float64 noisy feet decide as the reference's float32 ones wherever the margin allows
    lab = rep[..., 290:]
    sure = (g["noisy_speed_margin"] > 1e-4) & (g["noisy_height_margin"] > 1e-5)
    assert np.array_equal(lab[sure], g["noisy_contacts"][sure])
    assert 0.05 < float(g["noisy_contacts"].mean()) < 0.95  # both labels occur among the noisy feet


def test_fixture_holds_lock_rotations_and_headings_near_180():
    g = golden("windows_noise.npz")
    bp = g["param_body_pose"].reshape(-1, 21, 3).astype(np.float64)
    d_lock = wno.lock_distance(wno.quat_from_rotvec(bp[:, LOCK_JOINT]))
    d_near = wno.lock_distance(wno.quat_from_rotvec(bp[:, NEAR_JOINT]))
    assert d_lock.max() < 3e-8 and np.abs(d_near - 1e-3).max() < 1e-5  # both clear of scipy's 1e-7 threshold
    n_x = g["noise_body_pose"][..., LOCK_JOINT, 1]
    assert (g["noise_body_pose"][KEEP_LOCK_WINDOW][..., [LOCK_JOINT, NEAR_JOINT], 1] == 0).all()  # noisy angles at the lock
    assert (np.abs(np.delete(n_x, KEEP_LOCK_WINDOW, axis=0)) >= 2.0).all()  # the others move off it: the split shows
    heading = Rotation.from_rotvec(g["param_global_orient"]).as_euler('zxy')[:, 0]
    assert np.abs(np.abs(heading) - np.pi).min() < 0.05


def _lock_rotations(middle, n, seed):
    g = np.random.default_rng(seed)
    e = np.stack([g.uniform(-180, 180, n), np.full(n, middle), g.uniform(-180, 180, n)], -1)
    return Rotation.from_euler('zxy', e, degrees=True)


@pytest.mark.parametrize("middle", [90.0, -90.0, 90.0 - np.degrees(1e-3), -90.0 + np.degrees(1e-3), 30.0, -60.0])
def test_oracle_euler_matches_scipy(middle):
    rot = _lock_rotations(middle, 500, int(middle * 10) % 1000)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = rot.as_euler('zxy')
    got = wno.euler_zxy(rot.as_quat())
    assert np.abs(got - want).max() < 1e-12, middle
    if abs(middle) == 90.0:
        assert (got[:, 2] == 0).all() and (want[:, 2] == 0).all()  # scipy's rule at the lock: third angle zero


def test_oracle_euler_matches_scipy_on_random_rotations():
    rv = np.random.default_rng(5).standard_normal((20000, 3)) * 1.5
    want = Rotation.from_rotvec(rv).as_euler('zxy')
    got = wno.euler_zxy(wno.quat_from_rotvec(rv))
    assert np.abs(got - want).max() < 1e-12


@pytest.mark.parametrize("middle", [0.3, 90.0, -90.0])
def test_oracle_euler_wraps_as_scipy_at_180_degrees(middle):
    """First and third angles at and next to +-180 deg: the same values as scipy, +pi and -pi included (one turn is
    added or taken away only outside [-pi, pi])."""
    g = np.random.default_rng(7)
    e = np.stack([g.choice([180.0, -180.0, 179.999999, -179.999999, 0.0], 2000), np.full(2000, middle),
                  g.choice([180.0, -180.0, 0.0, 30.0], 2000)], -1)
    q = Rotation.from_euler('zxy', e, degrees=True).as_quat()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        want = Rotation.from_quat(q).as_euler('zxy')
    got = wno.euler_zxy(q)
    assert np.abs(got - want).max() < 1e-12
    assert (np.abs(want[:, 0]) == np.pi).any() or middle != 0.3


def _wrong_split(euler, shift=0.7):
    """euler_zxy with another (first, third) split of the same rotation at the lock: shift radians moved from the first
    angle to the third, with the sign that keeps the rotation."""
    def f(q):
        e = euler(q)
        lock = wno.lock_distance(q) <= wno.EULER_LOCK
        alt = e.copy()
        # at +90 deg Ry(c) Rx(90) Rz(a) depends on c - a only, at -90 deg on c + a
        alt[lock, 0] -= shift
        alt[lock, 2] -= np.sign(e[lock, 1]) * shift
        if lock.any():
            r0 = Rotation.from_euler('zxy', e[lock]).as_matrix()
            r1 = Rotation.from_euler('zxy', alt[lock]).as_matrix()
            assert np.abs(r0 - r1).max() < 1e-6, "the other split is not the same rotation"
        return alt
    return f


def test_fixture_pins_the_split_at_the_lock(monkeypatch):
    """The fixture's lock joint has middle-angle noise, so a different (first, third) split at the lock -- the same
    clean rotation -- gives a noisy rotation about shift * |n_x| away: far outside the 1e-4 the GPU test allows the
    device's noisy parameters against the fixture.  With the noise-free middle angle (window KEEP_LOCK_WINDOW) the split
    does not show."""
    g = golden("windows_noise.npz")
    L, overlap, lengths, params, joints, noise = noise_case(g)
    model = synthetic.smplx_like_model(0)
    want = g["noisy_param_body_pose"].reshape(-1, L, 21, 3)[:, :, LOCK_JOINT]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        right = wno.encode_noisy(params, joints, lengths, noise, model, L, overlap)[0]['body_pose']
        monkeypatch.setattr(wno, "euler_zxy", _wrong_split(wno.euler_zxy))
        wrong = wno.encode_noisy(params, joints, lengths, noise, model, L, overlap)[0]['body_pose']
    right, wrong = right.reshape(-1, L, 21, 3)[:, :, LOCK_JOINT], wrong.reshape(-1, L, 21, 3)[:, :, LOCK_JOINT]
    assert np.abs(right - want).max() < 1e-6
    moved = np.abs(wrong - want).max(axis=(1, 2))
    for w in range(len(moved)):
        if w == KEEP_LOCK_WINDOW:
            assert moved[w] < 1e-6, moved
        else:
            assert moved[w] > 1e-2, moved


def test_input_noise_refusals_without_a_device():
    z = lambda *s: torch.zeros(*s)
    with pytest.raises(RohmB200Error, match="CUDA"):
        windows.InputNoise.given(z(2, 24, 3), z(2, 24, 10), z(2, 24, 3), z(2, 24, 21, 3))
    with pytest.raises(RohmB200Error, match="torch tensor"):
        windows.InputNoise.given(np.zeros((2, 24, 3)), z(2, 24, 10), z(2, 24, 3), z(2, 24, 21, 3))
    with pytest.raises(RohmB200Error, match="list or tuple"):
        windows.InputNoise.drawn(torch.Generator())
    for bad in (dict(std_transl=-0.1), dict(std_betas=float('nan')), dict(std_body_rot='3'), dict(std_global_rot=True)):
        with pytest.raises(RohmB200Error, match="standard deviation"):
            windows.InputNoise.drawn([], **bad)
    p = {k: torch.zeros(145, w) for k, w in windows.PARAMS}
    with pytest.raises(RohmB200Error, match="InputNoise"):
        windows.encode_joints(p, torch.zeros(145, 22, 3), [145], None, None, noise="noise")
    with pytest.raises(RohmB200Error, match="body_model"):
        windows.encode_joints(p, torch.zeros(145, 22, 3), [145], None, None, noise=windows.InputNoise.drawn([]))
