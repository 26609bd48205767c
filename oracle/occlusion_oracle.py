"""float64 numpy restatement of the joint occlusion masks (rohm_b200/csrc/occlusion.cu, DESIGN §4.17): cv2.projectPoints,
the pixel-centre ray test, the scene depth map by per-triangle screen boxes, and the mask rule of
utils/get_occlusion_mask.py with numpy 1.22's float64 comparison.  Every elementwise operation is one IEEE-rounded numpy
ufunc in the order the kernels use, so the kernels' results are these bits."""
import numpy as np

JOINTS = 25
THRESHOLD = 0.1


def project(points, camera_mtx, dist):
    """cv2.projectPoints(points, 0, 0, camera_mtx, dist) for float32 points [..., 3] -> float32 [..., 2], in OpenCV's
    order of operations (the identity rotation's zero products included)."""
    P = np.asarray(points, np.float32).astype(np.float64)
    K = np.asarray(camera_mtx, np.float64).reshape(3, 3)
    k = np.zeros(14)
    d = np.asarray(dist, np.float64).reshape(-1)
    k[:d.size] = d
    X, Y, Z = P[..., 0], P[..., 1], P[..., 2]
    with np.errstate(all="ignore"):
        x = ((1.0 * X + 0.0 * Y) + 0.0 * Z) + 0.0
        y = ((0.0 * X + 1.0 * Y) + 0.0 * Z) + 0.0
        z = ((0.0 * X + 0.0 * Y) + 1.0 * Z) + 0.0
        z = np.where(z != 0.0, 1.0 / np.where(z != 0.0, z, 1.0), 1.0)
        x, y = x * z, y * z
        r2 = x * x + y * y
        r4 = r2 * r2
        r6 = r4 * r2
        a1 = (2.0 * x) * y
        a2 = r2 + (2.0 * x) * x
        a3 = r2 + (2.0 * y) * y
        cdist = ((1.0 + k[0] * r2) + k[1] * r4) + k[4] * r6
        icdist2 = 1.0 / (((1.0 + k[5] * r2) + k[6] * r4) + k[7] * r6)
        xd0 = (((x * cdist) * icdist2 + k[2] * a1) + k[3] * a2 + k[8] * r2) + k[9] * r4
        yd0 = (((y * cdist) * icdist2 + k[2] * a3) + k[3] * a1 + k[10] * r2) + k[11] * r4
        t0 = (1.0 * xd0 + 0.0 * yd0) + 0.0 * 1.0
        t1 = (0.0 * xd0 + 1.0 * yd0) + 0.0 * 1.0
        t2 = (0.0 * xd0 + 0.0 * yd0) + 1.0 * 1.0
        ip = np.where(t2 != 0.0, 1.0 / np.where(t2 != 0.0, t2, 1.0), 1.0)
        u = (ip * t0) * K[0, 0] + K[0, 2]
        v = (ip * t1) * K[1, 1] + K[1, 2]
    return np.stack([u, v], axis=-1).astype(np.float32)


def pixels(uv, size):
    """float32 coordinates [..., 2] -> (pixel int32 [..., 2], on_screen bool [...]).  numpy's astype(int) truncates toward
    zero; a coordinate that is non-finite or beyond int64 becomes INT64_MIN on x86 and is off screen.  So a joint is on
    screen iff -1 < u < W and -1 < v < H.  The int32 pixel is the truncation where finite and below 2^31 in magnitude,
    INT32_MIN elsewhere."""
    uv = np.asarray(uv, np.float32)
    W, H = size
    with np.errstate(invalid="ignore"):
        ok = np.isfinite(uv) & (np.abs(uv) < np.float32(2147483648.0))
        pix = np.where(ok, np.trunc(np.where(ok, uv, 0)), np.iinfo(np.int32).min).astype(np.int32)
        on = (uv[..., 0] > -1) & (uv[..., 0] < W) & (uv[..., 1] > -1) & (uv[..., 1] < H)
    return pix, on


def ray_dirs(px, py, intr):
    fx, fy, cx, cy = (float(v) for v in intr)
    return ((np.asarray(px, np.float64) + 0.5) - cx) / fx, ((np.asarray(py, np.float64) + 0.5) - cy) / fy


def ray_depth(dx, dy, v0, v1, v2, znear, zfar):
    """The kernels' Möller-Trumbore from the camera centre (broadcasting): (hit bool, z float64, NaN where missed)."""
    with np.errstate(all="ignore"):
        e1 = [v1[..., i] - v0[..., i] for i in range(3)]
        e2 = [v2[..., i] - v0[..., i] for i in range(3)]
        p = [dy * e2[2] - e2[1], e2[0] - dx * e2[2], dx * e2[1] - dy * e2[0]]
        det = (e1[0] * p[0] + e1[1] * p[1]) + e1[2] * p[2]
        s = [-v0[..., i] for i in range(3)]
        u = (s[0] * p[0] + s[1] * p[1]) + s[2] * p[2]
        q = [s[1] * e1[2] - s[2] * e1[1], s[2] * e1[0] - s[0] * e1[2], s[0] * e1[1] - s[1] * e1[0]]
        v = (dx * q[0] + dy * q[1]) + q[2]
        t = ((e2[0] * q[0] + e2[1] * q[1]) + e2[2] * q[2]) / det
        hit = (det > 0) & (u >= 0) & (v >= 0) & (u + v <= det) & (t >= znear) & (t <= zfar)
    return hit, np.where(hit, t, np.nan)


def screen_boxes(v0, v1, v2, intr, size, znear, zfar):
    """Conservative screen boxes of triangles [F, 3] x3 in the camera frame -> (x0, y0, x1, y1 int64 [F], valid [F]),
    as the kernels' screen_box: vertices with z >= znear and the znear crossings of the edges, projected, padded by one
    pixel, clipped to the viewport."""
    fx, fy, cx, cy = (float(v) for v in intr)
    W, H = size
    F = v0.shape[0]
    umin, vmin = np.full(F, np.inf), np.full(F, np.inf)
    umax, vmax = np.full(F, -np.inf), np.full(F, -np.inf)
    with np.errstate(all="ignore"):
        def take(x, y, z, m):
            u = fx * (x / z) + cx
            v = fy * (y / z) + cy
            umin[m], umax[m] = np.minimum(umin[m], u[m]), np.maximum(umax[m], u[m])
            vmin[m], vmax[m] = np.minimum(vmin[m], v[m]), np.maximum(vmax[m], v[m])

        for a in (v0, v1, v2):
            take(a[:, 0], a[:, 1], a[:, 2], a[:, 2] >= znear)
        for a, b in ((v0, v1), (v1, v2), (v2, v0)):
            m = (a[:, 2] < znear) != (b[:, 2] < znear)
            s = (znear - a[:, 2]) / (b[:, 2] - a[:, 2])
            take(a[:, 0] + (b[:, 0] - a[:, 0]) * s, a[:, 1] + (b[:, 1] - a[:, 1]) * s, np.full(F, znear), m)
        lx = np.maximum(np.floor(umin - 0.5) - 1.0, 0.0)
        hx = np.minimum(np.ceil(umax - 0.5) + 1.0, W - 1.0)
        ly = np.maximum(np.floor(vmin - 0.5) - 1.0, 0.0)
        hy = np.minimum(np.ceil(vmax - 0.5) + 1.0, H - 1.0)
        finite = np.isfinite(v0).all(1) & np.isfinite(v1).all(1) & np.isfinite(v2).all(1)
        z = np.stack([v0[:, 2], v1[:, 2], v2[:, 2]], 1)
        valid = finite & ~(z < znear).all(1) & ~(z > zfar).all(1) & (lx <= hx) & (ly <= hy)
    cast = lambda a: np.where(valid, a, 0).astype(np.int64)
    return cast(lx), cast(ly), cast(hx), cast(hy), valid


def to_camera(vertices, world2cam):
    """float32 world vertices [V,3] -> float64 camera frame: ((R0 X + R1 Y) + R2 Z) + t per row."""
    X = np.asarray(vertices, np.float32).astype(np.float64)
    M = np.asarray(world2cam, np.float64).reshape(3, 4)
    return np.stack([((M[r, 0] * X[:, 0] + M[r, 1] * X[:, 1]) + M[r, 2] * X[:, 2]) + M[r, 3] for r in range(3)], 1)


def scene_depth(vertices, faces, world2cam, intr, size, znear=0.05, zfar=100.0, pairs_per_chunk=1 << 22):
    """The depth map [H, W] float32 of rohm_scene_depth: per pixel the smallest accepted ray_depth over the triangles
    whose screen box holds it, rounded to float32; 0 without a hit."""
    W, H = size
    cv = to_camera(vertices, world2cam)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    v0, v1, v2 = cv[f[:, 0]], cv[f[:, 1]], cv[f[:, 2]]
    x0, y0, x1, y1, valid = screen_boxes(v0, v1, v2, intr, size, znear, zfar)
    idx = np.nonzero(valid)[0]
    bw, bh = (x1 - x0 + 1)[idx], (y1 - y0 + 1)[idx]
    area = bw * bh
    best = np.full(W * H, np.inf)
    ends = np.cumsum(area)
    lo = 0
    while lo < idx.size:
        hi = int(np.searchsorted(ends, (ends[lo - 1] if lo else 0) + pairs_per_chunk, side='right'))
        hi = max(hi, lo + 1)
        tri = np.repeat(np.arange(lo, hi), area[lo:hi])
        first = np.repeat(ends[lo:hi] - area[lo:hi], area[lo:hi])
        p = np.arange(first.size) + (ends[lo - 1] if lo else 0) - first
        x = x0[idx[tri]] + p % bw[tri]
        y = y0[idx[tri]] + p // bw[tri]
        dx, dy = ray_dirs(x, y, intr)
        t = idx[tri]
        hit, z = ray_depth(dx, dy, v0[t], v1[t], v2[t], znear, zfar)
        np.minimum.at(best, (y * W + x)[hit], z[hit])
        lo = hi
    out = np.where(np.isfinite(best), best, 0.0).astype(np.float32)
    return out.reshape(H, W)


def mask_rule(depth_body, depth_scene, on_screen):
    """get_occlusion_mask.py:131-140: occluded (0) iff on screen, scene depth != 0 and float64(body - scene) > 0.1, the
    difference taken in float32 and compared in float64 (numpy 1.22's float32-scalar-vs-Python-float rule)."""
    db = np.asarray(depth_body, np.float32)
    ds = np.asarray(depth_scene, np.float32)
    diff = (db - ds).astype(np.float64)
    occluded = on_screen & (ds != 0) & (diff > THRESHOLD)
    return np.where(occluded, 0.0, 1.0).astype(np.float32)


def body_depths(joints25, verts, faces, pix, on_screen, intr, size, znear=0.05, zfar=100.0):
    """One frame: the body's depth [25] float32 at each on-screen joint's pixel (0 for a miss or off screen)."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    V = np.asarray(verts, np.float32).astype(np.float64)
    v0, v1, v2 = V[f[:, 0]], V[f[:, 1]], V[f[:, 2]]
    x0, y0, x1, y1, valid = screen_boxes(v0, v1, v2, intr, size, znear, zfar)
    out = np.zeros(JOINTS, np.float32)
    for j in np.nonzero(on_screen)[0]:
        x, y = int(pix[j, 0]), int(pix[j, 1])
        cand = np.nonzero(valid & (x0 <= x) & (x <= x1) & (y0 <= y) & (y <= y1))[0]
        if cand.size == 0:
            continue
        dx, dy = ray_dirs(x, y, intr)
        hit, z = ray_depth(dx, dy, v0[cand], v1[cand], v2[cand], znear, zfar)
        if hit.any():
            out[j] = np.float32(z[hit].min())
    return out


def joint_occlusion(joints, verts, faces, frame_rec, camera_mtx, dist, depth_maps, map_of_rec, intr, size, znear=0.05,
                    zfar=100.0):
    """rohm_joint_occlusion over N frames: joints [N, >=25, 3], verts [N, V, 3] float32 (camera frame), frame_rec [N],
    camera_mtx [R,3,3], dist [R, n], depth_maps [S, H, W], map_of_rec [R] -> (mask [N,25] float32, pixel [N,25,2] int32,
    depth_body [N,25], depth_scene [N,25])."""
    joints = np.asarray(joints, np.float32)
    N = joints.shape[0]
    W, H = size
    mask = np.ones((N, JOINTS), np.float32)
    pixel = np.zeros((N, JOINTS, 2), np.int32)
    db = np.zeros((N, JOINTS), np.float32)
    ds = np.zeros((N, JOINTS), np.float32)
    for n in range(N):
        r = int(frame_rec[n])
        uv = project(joints[n, :JOINTS], camera_mtx[r], dist[r])
        pix, on = pixels(uv, size)
        pixel[n] = pix
        db[n] = body_depths(joints[n, :JOINTS], verts[n], faces, pix, on, intr, size, znear, zfar)
        dmap = depth_maps[int(map_of_rec[r])]
        ds[n] = np.where(on, dmap[np.where(on, pix[:, 1], 0), np.where(on, pix[:, 0], 0)], 0).astype(np.float32)
        mask[n] = mask_rule(db[n], ds[n], on)
    return mask, pixel, db, ds
