"""GPU: the joint occlusion masks (rohm_b200.occlusion: rohm_scene_depth, rohm_joint_occlusion) against the float64
numpy restatement (oracle/occlusion_oracle.py) bit for bit, on synthetic scenes and bodies, at every branch of the mask
rule, and invariant to batching, order and chunking."""
import numpy as np
import pytest
import torch

from oracle import occlusion_oracle as oo
from rohm_b200 import occlusion, synthetic, windows
from rohm_b200._lib import RohmB200Error
from rohm_b200.body_model import BodyModel
from test_gpu_windows import _recording_params

pytestmark = pytest.mark.gpu

INTR = occlusion.PROX_RENDER_INTRINSICS
SIZE = occlusion.RENDER_SIZE
ZN, ZF = occlusion.ZNEAR, occlusion.ZFAR


def _bits(t):
    return t.contiguous().view(torch.int32).cpu().numpy()


def _front(V, F):
    """F re-wound so each triangle faces the camera (n . v0 < 0)."""
    a, b, c = V[F[:, 0]].astype(np.float64), V[F[:, 1]].astype(np.float64), V[F[:, 2]].astype(np.float64)
    back = (np.cross(b - a, c - a) * a).sum(1) > 0
    F = F.copy()
    F[back] = F[back][:, [0, 2, 1]]
    return F


def _rigid(seed):
    g = np.random.default_rng(seed)
    a, b = g.uniform(-0.4, 0.4, 2)
    Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    Rx = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]])
    M = np.eye(4)
    M[:3, :3] = Rz @ Rx
    M[:3, 3] = g.uniform(-2, 2, 3)
    return M


def scene(seed, intr=INTR, size=SIZE, n_small=4000):
    """(world vertices float32 [V,3], faces [F,3], cam2world [4,4]) of a synthetic scene, designed in the camera frame:
    sub-pixel triangles, triangles of a few to many pixels (both sides of the large-box threshold), a floor and walls,
    slivers and degenerate triangles, back faces, triangles straddling znear and zfar, coplanar overlapping pairs."""
    g = np.random.default_rng(seed)
    fx, fy, cx, cy = intr
    W, H = size
    Vs, Fs = [], []

    def add(tris, front=True):
        tris = np.asarray(tris, np.float64).reshape(-1, 3, 3)
        n = len(Vs) and sum(len(v) for v in Vs)
        F = np.arange(len(tris) * 3).reshape(-1, 3) + n
        V = tris.reshape(-1, 3)
        F = _front(V, F - n) + n
        if not front:
            F = F[:, [0, 2, 1]]
        Vs.append(V), Fs.append(F)

    def at(u, v, z):  # camera-frame point of pixel coordinate (u, v) at depth z
        return np.stack([(u - cx) / fx * z, (v - cy) / fy * z, z], -1)

    def blobs(n, px_size, zlo, zhi, front_share=0.5):
        c = np.stack([g.uniform(-20, W + 20, n), g.uniform(-20, H + 20, n)], -1)
        z = g.uniform(zlo, zhi, n)
        pts = c[:, None, :] + g.normal(0, px_size, (n, 3, 2))
        tris = at(pts[..., 0], pts[..., 1], np.repeat(z[:, None], 3, 1) + g.normal(0, 0.05, (n, 3)))
        keep = g.uniform(size=n) < front_share
        add(tris[keep]), add(tris[~keep], front=False)

    blobs(n_small, 0.3, 1.0, 8.0)                    # sub-pixel
    blobs(max(n_small // 40, 8), 12.0, 1.5, 8.0, 0.7)   # boxes of ~10^2 .. 10^3 pixels
    blobs(max(n_small // 200, 4), 40.0, 1.5, 8.0, 0.7)  # beyond the threshold
    # floor (y = 1.2 below the camera), back wall, a near wall over part of the view
    add([[[-30, 1.2, 0.3], [30, 1.2, 0.3], [30, 1.2, 60]], [[-30, 1.2, 0.3], [30, 1.2, 60], [-30, 1.2, 60]]])
    add([[[-40, -30, 9], [5, -30, 9], [5, 30, 9]], [[-40, -30, 9], [5, 30, 9], [-40, 30, 9]]])  # leaves the right open
    add([at(np.float64([W * 0.55, W * 0.95, W * 0.95]), np.float64([H * 0.1, H * 0.1, H * 0.9]), np.full(3, 2.8)),
         at(np.float64([W * 0.55, W * 0.95, W * 0.55]), np.float64([H * 0.1, H * 0.9, H * 0.9]), np.full(3, 2.8))])
    # slivers (1e-4 pixel wide, hundreds long) and degenerate triangles (collinear, repeated vertices)
    for i in range(20):
        u0, v0 = g.uniform(0, W), g.uniform(0, H)
        z = g.uniform(1, 5)
        add(at(np.float64([u0, u0 + 300, u0 + 150]), np.float64([v0, v0 + 200, v0 + 100 + 1e-4 * (i % 3)]), np.full(3, z)))
        add(at(np.float64([u0, u0, u0]), np.float64([v0, v0, v0 + 5]), np.full(3, z)))
    # straddling znear and zfar
    for i in range(12):
        u0, v0 = g.uniform(0, W), g.uniform(0, H)
        add(at(np.float64([u0, u0 + 200, u0 + 40]), np.float64([v0, v0 + 30, v0 + 180]), np.float64([0.01, 0.2, 0.06])))
        add(at(np.float64([u0, u0 + 90, u0 + 20]), np.float64([v0, v0 + 10, v0 + 80]), np.float64([70, 140, 99.99])))
    # coplanar overlapping pairs
    for i in range(10):
        u0, v0 = g.uniform(0, W), g.uniform(0, H)
        z = g.uniform(2, 6)
        add(at(np.float64([u0, u0 + 60, u0]), np.float64([v0, v0, v0 + 60]), np.full(3, z)))
        add(at(np.float64([u0 + 10, u0 + 70, u0 + 10]), np.float64([v0 + 5, v0 + 5, v0 + 65]), np.full(3, z)))
    Vc = np.concatenate(Vs)
    F = np.concatenate(Fs)
    c2w = _rigid(seed)
    Vw = (Vc @ c2w[:3, :3].T + c2w[:3, 3]).astype(np.float32)
    perm = g.permutation(len(F))
    return Vw, F[perm], c2w


@pytest.mark.parametrize("size,intr", [(SIZE, INTR), ((37, 23), (21.3, 20.7, 18.1, 11.6))])
def test_scene_depth_equals_the_oracle_on_every_pixel(cuda_device, size, intr):
    V, F, c2w = scene(3, intr, size, n_small=4000 if size == SIZE else 300)
    d0 = occlusion.scene_depth(torch.from_numpy(V).to(cuda_device), F, c2w, intr, size)
    d1 = occlusion.scene_depth(V, torch.from_numpy(F), c2w, intr, size)
    ref = oo.scene_depth(V, F, occlusion.world_to_camera(c2w), intr, size, ZN, ZF)
    assert tuple(d0.shape) == (size[1], size[0])
    assert np.array_equal(_bits(d0), _bits(d1)), "the depth map changed between two runs"
    got = d0.cpu().numpy()
    assert np.array_equal(got.view(np.int32), ref.view(np.int32)), \
        f"{np.count_nonzero(got != ref)} pixels differ; worst {np.abs(got - ref).max()}"
    drawn = ref > 0
    assert 0.3 < drawn.mean() < 1.0 and (ref[drawn] >= np.float32(ZN)).all() and (ref[drawn] <= np.float32(ZF)).all()


def test_scene_depth_refuses_bad_input(cuda_device):
    V, F, c2w = scene(1, n_small=10)
    with pytest.raises(RohmB200Error):
        occlusion.scene_depth(V, F + len(V), c2w)
    with pytest.raises(RohmB200Error):
        occlusion.scene_depth(V, F, np.full((4, 4), np.nan))
    with pytest.raises(RohmB200Error):
        occlusion.scene_depth(V[:, :2], F, c2w)


# ---------------------------------------------------------------------------------------------------- bodies
@pytest.fixture(scope="module")
def body(cuda_device):
    return BodyModel.create('', device=cuda_device, seed=0), synthetic.smplx_like_faces(0)


LENGTHS = (0, 1, 145, 700)
KS = np.array([[[1060.53, 0.0, 951.30], [0.0, 1060.38, 536.77], [0.0, 0.0, 1.0]],
               [[1012.0, 0.0, 990.5], [0.0, 1009.5, 520.25], [0.0, 0.0, 1.0]]])
DIST = np.array([[0.0437, -0.0597, -0.0011, 0.0007, 0.0210, 0.0, 0.0, 0.0],
                 [-0.021, 0.035, 0.0006, -0.0009, -0.011, 0.0013, -0.0021, 0.0041]])


def _params(lengths, dev, seed0=11):
    recs = [_recording_params(n, seed0 + i) for i, n in enumerate(lengths)]
    p = {k: np.concatenate([r[k] for r in recs]).astype(np.float32) for k in recs[0]}
    p['transl'] = (p['transl'] * np.float32([0.4, 0.25, 0.0]) + np.float32([0.0, -0.2, 3.0])).astype(np.float32)
    # a few frames far off to the side, and one with the body behind the camera
    p['transl'][::97, 0] += 4.0
    p['transl'][5::211, 2] = -2.0
    return {k: torch.from_numpy(v).to(dev) for k, v in p.items()}


@pytest.fixture(scope="module")
def maps(cuda_device):
    out = []
    for s in (5, 6):
        V, F, c2w = scene(s, n_small=1500)
        out.append(occlusion.scene_depth(V, F, c2w))
    return torch.stack(out)


def _case(lengths, order=None):
    R = len(lengths)
    cams = [i % 2 for i in range(R)] if order is None else [order[i] % 2 for i in range(R)]
    return np.asarray(cams), KS[cams], DIST[cams]


def test_joint_mask_equals_the_oracle_with_the_synthetic_body(cuda_device, body, maps):
    model, faces = body
    p = _params(LENGTHS, cuda_device)
    map_of, K, k = _case(LENGTHS)
    got = occlusion.joint_mask(model, faces, p, LENGTHS, maps, map_of, K, k, details=True,
                               chunk_frames=sum(LENGTHS))
    out = model(**p, return_verts=True)
    frame_rec = np.repeat(np.arange(len(LENGTHS)), LENGTHS)
    mask, pix, db, ds = oo.joint_occlusion(out.joints.cpu().numpy(), out.vertices.cpu().numpy(), faces, frame_rec, K, k,
                                           maps.cpu().numpy(), map_of, INTR, SIZE, ZN, ZF)
    assert np.array_equal(got['pixel'].cpu().numpy(), pix)
    assert np.array_equal(_bits(got['depth_body']), db.view(np.int32))
    assert np.array_equal(_bits(got['depth_scene']), ds.view(np.int32))
    assert np.array_equal(_bits(got['mask']), mask.view(np.int32))
    # the rule's branches all occur: occluded, visible over the scene, body misses, off screen
    on = (pix[..., 0] >= 0) & (pix[..., 0] < SIZE[0]) & (pix[..., 1] >= 0) & (pix[..., 1] < SIZE[1])
    assert (mask == 0).sum() > 100 and (mask[on] == 1).sum() > 100
    assert ((db == 0) & on).any() and (~on).any()
    assert np.array_equal(got['mask'].cpu().numpy(), occlusion.joint_mask(model, faces, p, LENGTHS, maps, map_of, K,
                                                                          k).cpu().numpy())


def test_each_recording_alone_batched_reordered_and_chunked(cuda_device, body, maps):
    model, faces = body
    p = _params(LENGTHS, cuda_device)
    map_of, K, k = _case(LENGTHS)
    full = occlusion.joint_mask(model, faces, p, LENGTHS, maps, map_of, K, k, details=True, chunk_frames=256)
    for chunk in (7, 1000):
        other = occlusion.joint_mask(model, faces, p, LENGTHS, maps, map_of, K, k, details=True, chunk_frames=chunk)
        for key in full:
            assert torch.equal(full[key], other[key]), (chunk, key)
    off = np.concatenate([[0], np.cumsum(LENGTHS)])
    rows = lambda r: slice(int(off[r]), int(off[r + 1]))
    for r in range(len(LENGTHS)):
        alone = occlusion.joint_mask(model, faces, {a: b[rows(r)] for a, b in p.items()}, (LENGTHS[r],), maps,
                                     map_of[r:r + 1], K[r:r + 1], k[r:r + 1], chunk_frames=97)
        assert torch.equal(alone, full['mask'][rows(r)]), r
    order = [3, 1, 0, 2]
    pr = {a: torch.cat([b[rows(r)] for r in order]) for a, b in p.items()}
    re = occlusion.joint_mask(model, faces, pr, [LENGTHS[r] for r in order], maps, map_of[order], K[order], k[order])
    lens = [LENGTHS[r] for r in order]
    roff = np.concatenate([[0], np.cumsum(lens)])
    for i, r in enumerate(order):
        assert torch.equal(re[int(roff[i]):int(roff[i + 1])], full['mask'][rows(r)]), r


def _cube(lo, hi):
    """A closed box [lo, hi] with outward-facing triangles (front-facing from outside)."""
    c = np.array([[x, y, z] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])], np.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    F = np.array([[q[0], q[1], q[2]] for q in quads] + [[q[0], q[2], q[3]] for q in quads])
    a, b, d = c[F[:, 0]].astype(np.float64), c[F[:, 1]].astype(np.float64), c[F[:, 2]].astype(np.float64)
    inward = (np.cross(b - a, d - a) * ((a + b + d) / 3 - (np.asarray(lo) + np.asarray(hi)) / 2)).sum(1) < 0
    F[inward] = F[inward][:, [0, 2, 1]]
    return c, F


def test_hand_built_meshes_hit_every_branch_of_the_rule(cuda_device):
    # the body's front face at zf = 2^-10 + f32(0.1); scene depths 2^-10 -+ 2^-27 and 2^-10 put the float32 difference
    # one ulp above, exactly at and one ulp below f32(0.1), where numpy 1.22's float64 comparison decides
    intr, size = (128.0, 128.0, 0.5, 0.5), (400, 300)
    base = np.float32(2.0 ** -10)
    zf = np.float32(base + np.float32(0.1))
    ulp = np.float32(2.0 ** -27)
    N = 4
    verts, joints = [], np.zeros((N, 55, 3), np.float32)
    scene_map = np.zeros((1, size[1], size[0]), np.float32)
    cases = [base - ulp, base, base + ulp, 0.0, 0.5, 'nan', 'off', 'behind']
    for f in range(N):
        lo, hi = (-0.05, -0.05, float(zf)), (0.3, 0.3, float(zf) + 1.0)
        if f == 3:  # the body far to the side: every on-screen joint misses it
            lo, hi = (5.0, -0.05, float(zf)), (6.0, 0.3, float(zf) + 1.0)
        V, F = _cube(lo, hi)
        verts.append(V)
        for j in range(25):
            px, py = 10 + 14 * j, 10 + 60 * f
            Z = np.float32(0.2)
            joints[f, j] = [(px + 0.25 - 0.5) / 128 * Z, (py + 0.25 - 0.5) / 128 * Z, Z]
            c = cases[j % len(cases)]
            if c == 'nan':
                joints[f, j, 0] = np.nan
            elif c == 'off':
                joints[f, j, 0] = 2.0
            elif c == 'behind':
                joints[f, j, 2] = -0.2
            else:
                scene_map[0, py, px] = c
    J = torch.from_numpy(joints).to(cuda_device)
    Vt = torch.from_numpy(np.stack(verts)).to(cuda_device)
    K = np.array([[[128.0, 0, 0.5], [0, 128.0, 0.5], [0, 0, 1]]])
    maps_t = torch.from_numpy(scene_map).to(cuda_device)
    got = occlusion.joint_mask_from_meshes(J, Vt, F, (N,), maps_t, [0], K, np.zeros((1, 4)), intr, size, details=True)
    mask, pix, db, ds = oo.joint_occlusion(joints, np.stack(verts), F, np.zeros(N, int), K, np.zeros((1, 4)), scene_map,
                                           [0], intr, size, ZN, ZF)
    assert np.array_equal(got['pixel'].cpu().numpy(), pix)
    assert np.array_equal(_bits(got['depth_body']), db.view(np.int32))
    assert np.array_equal(_bits(got['depth_scene']), ds.view(np.int32))
    assert np.array_equal(_bits(got['mask']), mask.view(np.int32))
    m = got['mask'].cpu().numpy()
    dbg = got['depth_body'].cpu().numpy()
    for f in range(3):
        for j in range(25):
            c = cases[j % len(cases)]
            if c == 'behind':
                continue
            if not isinstance(c, str):
                assert dbg[f, j] == zf, (f, j)
            want = 0.0 if (not isinstance(c, str) and c != 0.0 and c < base + ulp) else 1.0
            assert m[f, j] == want, (f, j, c)
    assert (m[3] == 1.0).all() and (dbg[3] == 0.0).all()
    assert pix[0, 5, 0] == np.iinfo(np.int32).min  # the NaN joint


def test_joint_mask_feeds_encode_video(cuda_device, body, maps):
    model, faces = body
    lengths = (150, 290)
    p = _params(lengths, cuda_device, seed0=40)
    map_of, K, k = _case(lengths)
    dm = occlusion.joint_mask(model, faces, p, lengths, maps, map_of, K, k)
    out = model(**p, return_verts=True)
    ref, _, _, _ = oo.joint_occlusion(out.joints.cpu().numpy(), out.vertices.cpu().numpy(), faces,
                                      np.repeat(np.arange(2), lengths), K, k, maps.cpu().numpy(), map_of, INTR, SIZE,
                                      ZN, ZF)
    assert (ref == 0).any()
    R, N = len(lengths), sum(lengths)
    gk = np.random.default_rng(5)
    kp = np.concatenate([gk.uniform(-200, 2100, (N, 25, 1)), gk.uniform(-100, 1200, (N, 25, 1)),
                         gk.uniform(0, 1, (N, 25, 1))], -1).astype(np.float32)
    ds_p = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_t = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    kw = dict(cam2world=np.repeat(np.eye(4)[None], R, 0), focal_length=KS[map_of][:, [0, 1], [0, 1]],
              camera_center=KS[map_of][:, [0, 1], [2, 2]], camera_mtx=K, dist=k,
              keypoints=torch.from_numpy(kp).to(cuda_device), pose_dataset=ds_p, traj_dataset=ds_t)
    a = windows.encode_video(model, p, lengths, 'prox', depth_mask=dm, **kw)
    b = windows.encode_video(model, p, lengths, 'prox', depth_mask=torch.from_numpy(ref).to(cuda_device), **kw)
    for x, y in zip(a[:2], b[:2]):
        assert x.keys() == y.keys()
        for key in x:
            if isinstance(x[key], dict):
                assert all(torch.equal(x[key][s], y[key][s]) for s in x[key]), key
            else:
                assert torch.equal(x[key], y[key]), key
    assert (a[1]['mask_joint_vis'] == 0).any()


def test_joint_mask_refuses_bad_input(cuda_device, body, maps):
    model, faces = body
    p = _params((3,), cuda_device)
    args = lambda **o: dict(dict(params=p, lengths=(3,), depth_maps=maps, map_of_recording=[0], camera_mtx=KS[:1],
                                 dist=DIST[:1]), **o)
    for bad in (dict(dist=DIST[:1, :6]), dict(map_of_recording=[2]), dict(camera_mtx=np.full((1, 3, 3), np.inf)),
                dict(lengths=(4,)), dict(depth_maps=maps[:, :10])):
        with pytest.raises(RohmB200Error):
            occlusion.joint_mask(model, faces, **args(**bad))
    with pytest.raises(RohmB200Error):
        occlusion.joint_mask(model, faces + 20000, **args())
