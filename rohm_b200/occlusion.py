"""The PROX joint occlusion masks (the reference's utils/get_occlusion_mask.py, DESIGN §4.17) on the device.

``scene_depth`` renders a scene mesh's depth map once per camera (rohm_scene_depth); ``joint_mask`` poses the body of
every frame of R recordings with the LBS kernels, projects its first 25 joints with the recording's colour camera as
cv2.projectPoints does and marks a joint occluded (0) where the scene at its pixel lies more than 0.1 m in front of the
body (rohm_joint_occlusion).  The result is the [N,25] ``mask_joint.npy`` of the reference and goes straight into
``windows.encode_video(depth_mask=...)``.

Both passes test only pixel-centre rays: depth is the smallest z in [ZNEAR, ZFAR] of a front-facing triangle hit by
the ray through the pixel's centre (edges included), in float64, rounded to float32.  ``read_ply`` and
``color_frames`` are the file side of tools/occlusion_masks.py, which writes the masks of a PROX layout.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib, glue
from ._lib import RohmB200Error
from .windows import DIST_LENGTHS, PARAMS

PROX_RENDER_INTRINSICS = (1060.53, 1060.38, 951.30, 536.77)  # fx, fy, cx, cy of the reference's IntrinsicsCamera
RENDER_SIZE = (1920, 1080)  # width, height
ZNEAR, ZFAR = 0.05, 100.0  # pyrender's defaults
JOINTS = 25
DEFAULT_CHUNK_FRAMES = 1024  # frames posed per LBS call: about 125 KB of vertices each


def _camera(intrinsics, size, name):
    try:
        fx, fy, cx, cy = (float(v) for v in intrinsics)
        W, H = (int(v) for v in size)
    except (TypeError, ValueError):
        raise RohmB200Error(f"{name}: intrinsics must be (fx, fy, cx, cy) and size (width, height)") from None
    if not all(np.isfinite((fx, fy, cx, cy))) or fx == 0 or fy == 0 or W <= 0 or H <= 0:
        raise RohmB200Error(f"{name}: intrinsics {intrinsics} and size {size} must be finite, fx, fy != 0, size > 0")
    return (fx, fy, cx, cy), (W, H)


def _host64(v, name, shape):
    a = v.detach().cpu().double().numpy() if torch.is_tensor(v) else np.asarray(v, dtype=np.float64)
    if a.ndim != len(shape) or any(w is not None and a.shape[i] != w for i, w in enumerate(shape)):
        want = ", ".join("n" if w is None else str(w) for w in shape)
        raise RohmB200Error(f"{name} must be [{want}], got {tuple(a.shape)}")
    if not np.isfinite(a).all():
        raise RohmB200Error(f"{name} holds a non-finite value")
    return a


def _faces_on(faces, n_verts, dev, name):
    """faces [F,3] as int32 on dev, every index in [0, n_verts)."""
    f = faces if torch.is_tensor(faces) else torch.from_numpy(np.ascontiguousarray(faces))
    if f.dim() != 2 or f.shape[1] != 3 or f.dtype.is_floating_point or f.dtype == torch.bool:
        raise RohmB200Error(f"{name}: faces must be an integer [F,3] array, got {tuple(f.shape)} {f.dtype}")
    if f.numel() and (int(f.min()) < 0 or int(f.max()) >= n_verts):
        raise RohmB200Error(f"{name}: face indices must lie in [0, {n_verts}), got [{int(f.min())}, {int(f.max())}]")
    return f.to(device=dev, dtype=torch.int32).contiguous()


def world_to_camera(cam2world):
    """The [3,4] float64 world -> camera map of a [4,4] camera -> world pose (numpy's inverse, as the reference
    applies inv(cam2world) to the scene)."""
    return np.ascontiguousarray(np.linalg.inv(_host64(cam2world, "occlusion: cam2world", (4, 4)))[:3])


def scene_depth(vertices, faces, cam2world, intrinsics=PROX_RENDER_INTRINSICS, size=RENDER_SIZE):
    """The depth map of a scene mesh seen by the render camera: vertices [V,3] in the world frame (any float array or
    tensor; CUDA tensors keep their device), faces [F,3], cam2world [4,4] -> CUDA float32 [H, W], 0 where nothing is
    hit.  Bit-deterministic."""
    (fx, fy, cx, cy), (W, H) = _camera(intrinsics, size, "occlusion.scene_depth")
    dev = vertices.device if torch.is_tensor(vertices) and vertices.is_cuda else \
        torch.device('cuda', torch.cuda.current_device())
    v = vertices if torch.is_tensor(vertices) else torch.from_numpy(np.asarray(vertices, np.float32))
    if v.dim() != 2 or v.shape[1] != 3:
        raise RohmB200Error(f"occlusion.scene_depth: vertices must be [V,3], got {tuple(v.shape)}")
    v = v.to(device=dev, dtype=torch.float32).contiguous()
    f = _faces_on(faces, v.shape[0], dev, "occlusion.scene_depth")
    w2c = world_to_camera(cam2world)
    lib, ctx = _lib.load(), _lib.ctx(dev.index)
    nbytes = lib.rohm_scene_depth_workspace_bytes(v.shape[0], f.shape[0], W, H)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    depth = torch.empty(H, W, dtype=torch.float32, device=dev)
    _lib.check(lib.rohm_scene_depth(ctx, glue._p(v), v.shape[0], glue._p(f), f.shape[0], w2c.ctypes.data_as(C.c_void_p),
                                    fx, fy, cx, cy, W, H, ZNEAR, ZFAR, glue._p(ws), nbytes, glue._p(depth), glue._stream(dev)), ctx)
    return depth


class _Cameras:
    """The per-recording inputs of rohm_joint_occlusion on one device, checked."""

    def __init__(self, R, depth_maps, map_of_recording, camera_mtx, dist, intrinsics, size, dev, name):
        self.intr, self.size = _camera(intrinsics, size, name)
        W, H = self.size
        K = _host64(camera_mtx, f"{name}: camera_mtx", (R, 3, 3))
        k = _host64(dist, f"{name}: dist", (R, None))
        if k.shape[1] not in DIST_LENGTHS:
            raise RohmB200Error(f"{name}: dist must hold {DIST_LENGTHS} coefficients per recording, got {k.shape[1]}")
        kpad = np.zeros((R, 14))
        kpad[:, :k.shape[1]] = k
        if not torch.is_tensor(depth_maps) or depth_maps.device != dev:
            raise RohmB200Error(f"{name}: depth_maps must be a CUDA tensor on {dev} (scene_depth's maps)")
        maps = depth_maps.unsqueeze(0) if depth_maps.dim() == 2 else depth_maps
        if maps.dim() != 3 or tuple(maps.shape[1:]) != (H, W):
            raise RohmB200Error(f"{name}: depth_maps must be [S, {H}, {W}], got {tuple(depth_maps.shape)}")
        m = np.asarray(map_of_recording, dtype=np.int64).reshape(-1)
        if m.shape[0] != R or (R and (m.min() < 0 or m.max() >= maps.shape[0])):
            raise RohmB200Error(f"{name}: map_of_recording must hold one index in [0, {maps.shape[0]}) per recording "
                                f"({R}), got {m.tolist()}")
        self.maps = maps.to(torch.float32).contiguous()
        self.K = torch.from_numpy(np.ascontiguousarray(K.reshape(R, 9))).to(dev)
        self.k = torch.from_numpy(kpad).to(dev)
        self.map_idx = torch.from_numpy(m.astype(np.int32)).to(dev)


def _outputs(N, dev, details):
    mask = torch.empty(N, JOINTS, dtype=torch.float32, device=dev)
    if not details:
        return {'mask': mask}
    return {'mask': mask, 'pixel': torch.empty(N, JOINTS, 2, dtype=torch.int32, device=dev),
            'depth_body': torch.empty(N, JOINTS, dtype=torch.float32, device=dev),
            'depth_scene': torch.empty(N, JOINTS, dtype=torch.float32, device=dev)}


def _run(cams, joints, verts, faces, frame_rec, out, s, dev):
    """rohm_joint_occlusion for frames [s, s + n) of the outputs: joints [n, J>=25, 3], verts [n, V, 3] with dense rows
    at any row pitch."""
    n = joints.shape[0]
    if n == 0:
        return
    if joints.stride(2) != 1 or joints.stride(1) != 3 or joints.stride(0) != 3 * joints.shape[1]:
        joints = joints.contiguous()
    if verts.stride(2) != 1 or verts.stride(1) != 3:
        verts = verts.contiguous()
    (fx, fy, cx, cy), (W, H) = cams.intr, cams.size
    sl = lambda k: glue._p(out[k][s:s + n]) if k in out else glue._p(None)
    lib, ctx = _lib.load(), _lib.ctx(dev.index)
    _lib.check(lib.rohm_joint_occlusion(ctx, glue._p(joints), joints.shape[1], glue._p(verts), verts.stride(0),
                                        glue._p(faces), faces.shape[0], glue._p(frame_rec[s:s + n]), n, glue._p(cams.K),
                                        glue._p(cams.k), glue._p(cams.maps), glue._p(cams.map_idx), fx, fy, cx, cy, W, H,
                                        ZNEAR, ZFAR, sl('mask'), sl('pixel'), sl('depth_body'), sl('depth_scene'),
                                        glue._stream(dev)), ctx)


def _lengths(lengths, name):
    lengths = tuple(int(n) for n in lengths)
    if not lengths or min(lengths) < 0:
        raise RohmB200Error(f"{name}: lengths must be one frame count >= 0 per recording, got {lengths}")
    return lengths


def _frame_rec(lengths, dev):
    return torch.from_numpy(np.repeat(np.arange(len(lengths)), lengths).astype(np.int32)).to(dev)


def joint_mask(body_model, faces, params, lengths, depth_maps, map_of_recording, camera_mtx, dist,
               intrinsics=PROX_RENDER_INTRINSICS, size=RENDER_SIZE, details=False, chunk_frames=DEFAULT_CHUNK_FRAMES):
    """The occlusion masks of R recordings packed frame after frame, as ``windows.encode_video`` takes them.

    body_model: ``BodyModel`` (or a module with its call convention), faces [F,3] its triangles (``body_model.load_faces``);
    params: the per-frame fits in each recording's camera frame (CUDA tensors global_orient [N,3], transl [N,3], betas
    [N,10], body_pose [N,63]), lengths: frames per recording; depth_maps [S,H,W] (``scene_depth``), map_of_recording [R]
    the map of each recording's scene; camera_mtx [R,3,3] and dist [R,n], n in (4, 5, 8): the colour camera of
    Color.json, which projects the joints (not the render intrinsics).  Returns CUDA float32 [N,25], 1 = visible; with
    details a dict of it ('mask') and, per joint, 'pixel' [N,25,2] int32 (INT32_MIN where not finite), 'depth_body' and
    'depth_scene' [N,25] (0 off screen).  Frames are posed chunk_frames at a time; a recording's masks do not depend on
    the chunking or on the other recordings of the call."""
    name = "occlusion.joint_mask"
    lengths = _lengths(lengths, name)
    R, N = len(lengths), sum(lengths)
    p = {}
    for key, width in PARAMS:
        t = glue._f32c(params[key], f"{name}: params['{key}']")
        if t.numel() != N * width:
            raise RohmB200Error(f"{name}: params['{key}'] must hold [{N}, {width}] (the packed recordings), got "
                                f"{tuple(t.shape)}")
        p[key] = t.reshape(N, width)
    dev = p['transl'].device
    if any(t.device != dev for t in p.values()):
        raise RohmB200Error(f"{name}: the parameters live on different devices")
    if isinstance(chunk_frames, bool) or not isinstance(chunk_frames, int) or chunk_frames < 1:
        raise RohmB200Error(f"{name}: chunk_frames must be an int >= 1, got {chunk_frames!r}")
    cams = _Cameras(R, depth_maps, map_of_recording, camera_mtx, dist, intrinsics, size, dev, name)
    f = _faces_on(faces, int(body_model.v_template.shape[0]), dev, name)
    frame_rec = _frame_rec(lengths, dev)
    out = _outputs(N, dev, details)
    for s in range(0, N, chunk_frames):
        e = min(N, s + chunk_frames)
        body = body_model(**{k: v[s:e] for k, v in p.items()}, return_verts=True)
        _run(cams, body.joints, body.vertices, f, frame_rec, out, s, dev)
    return out if details else out['mask']


def joint_mask_from_meshes(joints, vertices, faces, lengths, depth_maps, map_of_recording, camera_mtx, dist,
                           intrinsics=PROX_RENDER_INTRINSICS, size=RENDER_SIZE, details=False):
    """``joint_mask`` for bodies given as meshes: joints [N,J,3] (J >= 25; the first 25 count) and vertices [N,V,3]
    float32 CUDA tensors in each recording's camera frame, packed like lengths, faces [F,3] over the V vertices."""
    name = "occlusion.joint_mask_from_meshes"
    lengths = _lengths(lengths, name)
    R, N = len(lengths), sum(lengths)
    for t, nm, d in ((joints, "joints", None), (vertices, "vertices", None)):
        if not torch.is_tensor(t) or not t.is_cuda or t.dtype != torch.float32 or t.dim() != 3 or t.shape[0] != N or \
                t.shape[2] != 3:
            raise RohmB200Error(f"{name}: {nm} must be a float32 CUDA tensor [{N}, n, 3], got "
                                f"{tuple(getattr(t, 'shape', ()))}")
    if joints.shape[1] < JOINTS:
        raise RohmB200Error(f"{name}: joints must hold at least {JOINTS} joints per frame, got {joints.shape[1]}")
    dev = joints.device
    if vertices.device != dev:
        raise RohmB200Error(f"{name}: vertices live on {vertices.device}, joints on {dev}")
    cams = _Cameras(R, depth_maps, map_of_recording, camera_mtx, dist, intrinsics, size, dev, name)
    f = _faces_on(faces, vertices.shape[1], dev, name)
    out = _outputs(N, dev, details)
    _run(cams, joints, vertices, f, _frame_rec(lengths, dev), out, 0, dev)
    return out if details else out['mask']


# ------------------------------------------------------------------------------------------------------------ files
_PLY_TYPES = {'char': 'i1', 'int8': 'i1', 'uchar': 'u1', 'uint8': 'u1', 'short': 'i2', 'int16': 'i2', 'ushort': 'u2',
              'uint16': 'u2', 'int': 'i4', 'int32': 'i4', 'uint': 'u4', 'uint32': 'u4', 'float': 'f4', 'float32': 'f4',
              'double': 'f8', 'float64': 'f8'}


def read_ply(path):
    """(vertices float64 [V,3], faces int64 [F,3]) of a triangle-mesh PLY file, ascii or binary_little_endian: the
    vertex element's x, y, z (any scalar type) and the face element's one list property.  Other elements and
    properties are skipped; a face that is not a triangle is refused."""
    with open(path, 'rb') as fh:
        if fh.readline().strip() != b'ply':
            raise RohmB200Error(f"read_ply: {path} is not a PLY file")
        fmt, elements = None, []
        while True:
            line = fh.readline()
            if not line:
                raise RohmB200Error(f"read_ply: {path} ends inside its header")
            tok = line.decode('ascii', 'replace').split()
            if not tok or tok[0] in ('comment', 'obj_info'):
                continue
            if tok[0] == 'end_header':
                break
            if tok[0] == 'format':
                fmt = tok[1]
            elif tok[0] == 'element':
                elements.append((tok[1], int(tok[2]), []))
            elif tok[0] == 'property':
                if tok[1] == 'list':
                    elements[-1][2].append((tok[4], 'list', _PLY_TYPES[tok[2]], _PLY_TYPES[tok[3]]))
                else:
                    elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]]))
        if fmt not in ('ascii', 'binary_little_endian'):
            raise RohmB200Error(f"read_ply: {path}: format {fmt!r} is not ascii or binary_little_endian")
        body = fh.read()
    verts, faces = None, np.zeros((0, 3), np.int64)
    if fmt == 'ascii':
        lines = iter(body.decode('ascii').splitlines())
        for name, count, props in elements:
            rows = [next(lines).split() for _ in range(count)]
            if name == 'vertex':
                order = [next(i for i, p in enumerate(props) if p[0] == c) for c in 'xyz']
                verts = np.array([[float(r[i]) for i in order] for r in rows], np.float64).reshape(-1, 3)
            elif name == 'face':
                if any(int(r[0]) != 3 for r in rows):
                    raise RohmB200Error(f"read_ply: {path} has a face that is not a triangle")
                faces = np.array([[int(v) for v in r[1:4]] for r in rows], np.int64).reshape(-1, 3)
    else:
        pos = 0
        for name, count, props in elements:
            lists = [p for p in props if len(p) == 4]
            if not lists:
                dt = np.dtype([(p[0], '<' + p[1]) for p in props])
                arr = np.frombuffer(body, dt, count, pos)
                pos += dt.itemsize * count
                if name == 'vertex':
                    verts = np.stack([arr[c].astype(np.float64) for c in 'xyz'], 1)
                continue
            if name != 'face' or len(props) != 1:
                raise RohmB200Error(f"read_ply: {path}: element {name!r} with list properties is not supported")
            _, _, ct, it = lists[0]
            dt = np.dtype([('n', '<' + ct), ('i', '<' + it, (3,))])
            arr = np.frombuffer(body, dt, count, pos)
            if (arr['n'] != 3).any():
                raise RohmB200Error(f"read_ply: {path} has a face that is not a triangle")
            faces = arr['i'].astype(np.int64)
            pos += dt.itemsize * count
    if verts is None:
        raise RohmB200Error(f"read_ply: {path} has no vertex element")
    return verts, faces


def color_frames(names):
    """The frame names the reference script takes from a Color directory listing, in its order: sorted, '.png' files,
    or '.jpg' files that are not hidden (``endswith('.png') or endswith('.jpg') and not startswith('.')``), each
    without its 4-character extension (the results/<frame>/000.pkl folder name)."""
    return [n[:-4] for n in sorted(names) if n.endswith('.png') or n.endswith('.jpg') and not n.startswith('.')]
