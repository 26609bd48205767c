"""CPU: the joint occlusion restatement (oracle/occlusion_oracle.py) against cv2.projectPoints bit for bit, on
known-answer geometry, and at every edge of the mask rule; the PLY reader and the reference script's frame selection
(rohm_b200.occlusion)."""
import numpy as np
import pytest

from oracle import occlusion_oracle as oo
from rohm_b200 import occlusion

cv2 = pytest.importorskip("cv2")

PROX_K = np.array([[1060.53, 0.0, 951.30], [0.0, 1060.38, 536.77], [0.0, 0.0, 1.0]])
DISTS = {4: [0.0437, -0.0597, -0.0011, 0.0007], 5: [0.0437, -0.0597, -0.0011, 0.0007, 0.0210],
         8: [0.0437, -0.0597, -0.0011, 0.0007, 0.0210, 0.0013, -0.0021, 0.0041]}


def _points(rng, n):
    P = np.empty((n, 3), np.float32)
    P[:, 0] = rng.uniform(-2, 2, n)
    P[:, 1] = rng.uniform(-1.2, 1.2, n)
    P[:, 2] = rng.uniform(0.3, 6, n)
    P[: n // 20, 2] = 0.0                                    # OpenCV's 1/z -> 1 rule
    P[n // 20: n // 10, 2] *= -1                             # behind the camera
    # pixel borders without distortion: u = 1919, 1920 (and one ulp either side), v = 1079, 1080
    m = n // 10
    u = np.repeat(np.float64([1919.0, 1920.0, 0.0, -1.0]), -(-m // 4))[:m]
    z = P[n // 10: n // 10 + m, 2].astype(np.float64)
    P[n // 10: n // 10 + m, 0] = ((u - PROX_K[0, 2]) / PROX_K[0, 0] * z).astype(np.float32)
    v = np.repeat(np.float64([1079.0, 1080.0, 0.0, -1.0]), -(-m // 4))[:m]
    P[n // 10: n // 10 + m, 1] = ((v - PROX_K[1, 2]) / PROX_K[1, 1] * z).astype(np.float32)
    # the float32 neighbours of integers in the coordinates themselves
    k = slice(n // 5, n // 5 + m)
    P[k, 0] = np.nextafter(np.round(P[k, 0]), np.float32(np.inf) * rng.choice([-1, 1], m)).astype(np.float32)
    return P


@pytest.mark.parametrize("ncoef", [4, 5, 8])
def test_projection_equals_cv2_bit_for_bit(ncoef):
    rng = np.random.default_rng(ncoef)
    P = _points(rng, 100_000)
    for K, d in ((PROX_K, np.asarray(DISTS[ncoef])), (PROX_K, np.zeros(ncoef))):
        ref = cv2.projectPoints(P, np.zeros(3), np.zeros(3), K, d)[0].reshape(-1, 2)
        assert ref.dtype == np.float32
        ours = oo.project(P, K, d)
        assert np.array_equal(ours.view(np.uint32), ref.view(np.uint32)), np.count_nonzero(ours != ref)
    # pixels near the borders come out on both sides of them
    ref = oo.project(P, PROX_K, np.zeros(ncoef))
    for c, lim in ((0, 1920), (1, 1080)):
        assert (ref[:, c] == lim - 1).any() and (ref[:, c] == lim).any()


def test_projection_of_non_finite_points_is_nan():
    P = np.array([[np.nan, 0, 2], [0, np.inf, 2], [0, 0, -np.inf], [1, 1, 0]], np.float32)
    ours = oo.project(P, PROX_K, DISTS[5])
    ref = cv2.projectPoints(P, np.zeros(3), np.zeros(3), PROX_K, np.asarray(DISTS[5]))[0].reshape(-1, 2)
    assert np.array_equal(np.isnan(ours), np.isnan(ref)) and np.isnan(ours[:3]).all()
    assert np.array_equal(ours[3], ref[3])


# ---------------------------------------------------------------------------------------------------- geometry
INTR = (128.0, 128.0, 0.5, 0.5)  # pixel x's ray is (x / 128, y / 128, 1): exact dyadic geometry
SIZE = (40, 30)


def _quad(x0, x1, y0, y1, z, front=True):
    V = np.array([[x0, y0, z], [x1, y0, z], [x1, y1, z], [x0, y1, z]], np.float32)
    F = np.array([[0, 2, 1], [0, 3, 2]]) if front else np.array([[0, 1, 2], [0, 2, 3]])
    return V, F


I34 = np.hstack([np.eye(3), np.zeros((3, 1))])


def test_axis_aligned_quad_covers_exactly_the_predicted_pixel_centres():
    # at z = 2 pixel x's centre ray meets x = x / 64: edges at 4/64 .. 12/64 and 3/64 .. 9/64 pass through centres
    V, F = _quad(4 / 64, 12 / 64, 3 / 64, 9 / 64, 2.0)
    d = oo.scene_depth(V, F, I34, INTR, SIZE)
    want = np.zeros((SIZE[1], SIZE[0]), np.float32)
    want[3:10, 4:13] = 2.0
    assert np.array_equal(d, want)
    # each triangle alone includes the shared diagonal x - 4 = (y - 3) * 8 / 6 and the centres on it
    d0 = oo.scene_depth(V, F[:1], I34, INTR, SIZE)
    d1 = oo.scene_depth(V, F[1:], I34, INTR, SIZE)
    assert np.array_equal(np.maximum(d0, d1), want)
    both = (d0 > 0) & (d1 > 0)
    ys, xs = np.nonzero(both)
    assert both.sum() >= 2 and np.all((xs - 4) * 6 == (ys - 3) * 8)


def test_back_faces_and_quads_outside_the_clip_range_draw_nothing():
    V, F = _quad(4 / 64, 12 / 64, 3 / 64, 9 / 64, 2.0, front=False)
    assert not oo.scene_depth(V, F, I34, INTR, SIZE).any()
    for z in (150.0, 0.04):
        V, F = _quad(4 / 64 * z / 2, 12 / 64 * z / 2, 3 / 64 * z / 2, 9 / 64 * z / 2, z)
        assert not oo.scene_depth(V, F, I34, INTR, SIZE).any(), z


def test_a_quad_straddling_znear_is_cut_at_znear():
    # the plane z = 0.02 + 0.5 x over x in [0, 0.1] runs from z = 0.02 to 0.07 through znear = 0.05
    V = np.array([[0.0, -0.1, 0.02], [0.1, -0.1, 0.07], [0.1, 0.1, 0.07], [0.0, 0.1, 0.02]], np.float32)
    F = np.array([[0, 2, 1], [0, 3, 2]])
    d = oo.scene_depth(V, F, I34, INTR, (400, 300))
    drawn = d > 0
    assert drawn.any() and (d[drawn] >= np.float32(0.05)).all()
    # analytic depth along pixel centre rays: z = 0.02 + 0.5 (x / 128) z  ->  z = 0.02 / (1 - x / 256)
    ys, xs = np.nonzero(np.ones_like(drawn))
    with np.errstate(all="ignore"):
        z = 0.02 / (1 - xs / 256.0)
        inside = (xs < 256) & (xs / 128.0 * z <= 0.1) & (np.abs(ys / 128.0 * z) <= 0.1)
    clear = inside & (np.abs(z - 0.05) > 1e-6)
    assert np.array_equal(drawn.reshape(-1)[clear], (z >= 0.05)[clear])
    assert (drawn.reshape(-1) <= inside).all() and (inside & (z < 0.05)).any()


def test_screen_box_skips_degenerate_and_non_finite_triangles():
    v = np.array([[0.1, 0.1, 2.0]])
    x0, y0, x1, y1, ok = oo.screen_boxes(v, v, v, INTR, SIZE, 0.05, 100.0)
    assert ok.all() and x1[0] - x0[0] == 3 and y1[0] - y0[0] == 3  # u = 6.9: columns 5..8
    hit, _ = oo.ray_depth(0.05, 0.05, v, v, v, 0.05, 100.0)
    assert not hit.any()
    bad = np.array([[np.nan, 0.1, 2.0]])
    assert not oo.screen_boxes(bad, v, v, INTR, SIZE, 0.05, 100.0)[4].any()


# ---------------------------------------------------------------------------------------------------- mask rule
def test_a_difference_of_exactly_float32_point_one_is_occluded():
    ds = np.float32(2.0 ** -10)
    db = np.float32(ds + np.float32(0.1))
    assert db - ds == np.float32(0.1)
    below = np.nextafter(db, np.float32(0))
    m = oo.mask_rule([db, below], [ds, ds], np.array([True, True]))
    assert m.tolist() == [0.0, 1.0]
    # numpy 2 compares a float32 scalar with 0.1 in float32, where the exact difference would count as visible
    assert not (np.float32(0.1) > 0.1) and float(np.float32(0.1)) > 0.1


def test_scene_depth_zero_body_miss_and_off_screen_are_visible():
    on = np.array([True, True, False, True])
    m = oo.mask_rule([5.0, 0.0, 5.0, 5.0], [0.0, 2.0, 1.0, 1.0], on)
    assert m.tolist() == [1.0, 1.0, 1.0, 0.0]


def test_pixels_truncate_toward_zero_and_non_finite_coordinates_are_off_screen():
    uv = np.array([[-0.5, -0.999], [-1.0, 3.0], [1919.9, 1079.9], [1920.0, 5.0], [np.nan, 3.0], [3.0, np.inf],
                   [-np.inf, 2.0], [3e9, 1.0]], np.float32)
    pix, on = oo.pixels(uv, (1920, 1080))
    assert on.tolist() == [True, False, True, False, False, False, False, False]
    assert pix[0].tolist() == [0, 0] and pix[2].tolist() == [1919, 1079]
    i32min = np.iinfo(np.int32).min
    assert pix[4, 0] == i32min and pix[5, 1] == i32min and pix[6, 0] == i32min and pix[7, 0] == i32min
    # numpy's own astype(int) on x86 agrees on which are off screen
    with np.errstate(invalid="ignore"):
        ii = uv.astype(np.int64)
    ref = (ii[:, 0] >= 0) & (ii[:, 0] < 1920) & (ii[:, 1] >= 0) & (ii[:, 1] < 1080)
    assert np.array_equal(ref, on)


def test_joint_occlusion_oracle_on_a_body_behind_a_wall():
    # a body quad at z = 3 behind a scene wall at z = 2 (occluded), and one joint beside the wall (visible)
    V, F = _quad(-0.5, 0.5, -0.5, 0.5, 3.0)
    K = np.array([[128.0, 0, 0.5], [0, 128.0, 0.5], [0, 0, 1]])
    scene = np.zeros((1, 300, 400), np.float32)
    scene[0, :, :100] = 2.0
    J = np.zeros((1, 25, 3), np.float32)
    J[0, :, 2] = 3.0
    J[0, 1:, 0] = 0.3  # pixel 128 * 0.1 = 12.8 -> column 12 for joint 0, 12.8 + ... beyond the wall for the rest
    J[0, 1:, 0] = np.float32(3.0 * 150 / 128)  # column 150: no wall
    mask, pix, db, ds = oo.joint_occlusion(J, V[None], F, [0], K[None], np.zeros((1, 4)), scene, [0], INTR, (400, 300))
    assert pix[0, 0].tolist() == [0, 0] and mask[0, 0] == 0.0 and db[0, 0] == 3.0 and ds[0, 0] == 2.0
    assert (mask[0, 1:] == 1.0).all() and (ds[0, 1:] == 0.0).all()


# ---------------------------------------------------------------------------------------------------- files
def _write_ply(path, V, F, fmt, vtype, ctype="uchar", itype="int"):
    names = {"float": "f4", "double": "f8", "uchar": "u1", "int": "i4", "uint": "u4"}
    head = ["ply", f"format {fmt} 1.0", "comment test", f"element vertex {len(V)}", f"property {vtype} x",
            f"property {vtype} y", f"property {vtype} z", "property uchar red", f"element face {len(F)}",
            f"property list {ctype} {itype} vertex_indices", "end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode())
        if fmt == "ascii":
            for v in V:
                fh.write(f"{float(v[0])!r} {float(v[1])!r} {float(v[2])!r} 7\n".encode())
            for f in F:
                fh.write(f"3 {f[0]} {f[1]} {f[2]}\n".encode())
        else:
            vd = np.dtype([("x", "<" + names[vtype]), ("y", "<" + names[vtype]), ("z", "<" + names[vtype]),
                           ("r", "u1")])
            va = np.zeros(len(V), vd)
            va["x"], va["y"], va["z"], va["r"] = V[:, 0], V[:, 1], V[:, 2], 7
            fd = np.dtype([("n", "<" + names[ctype]), ("i", "<" + names[itype], (3,))])
            fa = np.zeros(len(F), fd)
            fa["n"], fa["i"] = 3, F
            fh.write(va.tobytes() + fa.tobytes())


@pytest.mark.parametrize("fmt,vtype,itype", [("ascii", "float", "int"), ("binary_little_endian", "float", "int"),
                                             ("binary_little_endian", "double", "uint"), ("ascii", "double", "int")])
def test_ply_reader_round_trips(tmp_path, fmt, vtype, itype):
    rng = np.random.default_rng(1)
    V = rng.normal(size=(57, 3)).astype(np.float32 if vtype == "float" else np.float64)
    F = rng.integers(0, 57, size=(91, 3))
    p = tmp_path / "scene.ply"
    _write_ply(p, V, F, fmt, vtype, itype=itype)
    v, f = occlusion.read_ply(str(p))
    assert np.array_equal(v, V.astype(np.float64)) and np.array_equal(f, F)


def test_ply_reader_refuses_non_triangles(tmp_path):
    p = tmp_path / "quad.ply"
    p.write_text("ply\nformat ascii 1.0\nelement vertex 4\nproperty float x\nproperty float y\nproperty float z\n"
                 "element face 1\nproperty list uchar int vertex_indices\nend_header\n0 0 0\n1 0 0\n1 1 0\n0 1 0\n"
                 "4 0 1 2 3\n")
    with pytest.raises(occlusion.RohmB200Error):
        occlusion.read_ply(str(p))


def test_frame_selection_matches_the_script_expression():
    listing = ["s001_frame_00002.jpg", "s001_frame_00001.jpg", ".s001_frame_00003.jpg", ".hidden.png", "notes.txt",
               "s001_frame_00010.png", "a.jpeg", "b.JPG", "._x.jpg", "c.png"]
    want = [f[0:-4] for f in sorted(listing)
            if f.endswith('.png') or f.endswith('.jpg') and not f.startswith('.')]
    assert occlusion.color_frames(listing) == want
    assert ".hidden" in want and ".s001_frame_00003" not in want
