"""SMPL-X-shaped body model container used when the third-party ``smplx`` package is not installed.

Holds the model tensors as buffers under smplx's own names (v_template, shapedirs, expr_dirs is folded into
shapedirs[..., 10:], posedirs, J_regressor, lbs_weights, parents) and evaluates joints / vertices with the CUDA
kernels of the library (rohm_fk22_* / rohm_lbs_forward).  See DESIGN.md for the provenance of the algorithm
(smplx==0.1.28, not vendored by the reference).
"""
import ctypes as C
import os

import numpy as np
import torch
import torch.nn as nn

from . import _lib, synthetic
from ._lib import RohmB200Error


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


class BodyOutput:
    """Mirror of smplx's output object: the attributes RoHM reads (``joints``, ``vertices``)."""

    def __init__(self, joints=None, vertices=None):
        self.joints = joints
        self.vertices = vertices


class BodyKernels:
    """One rohm_body handle (device copies of the model + per-call workspace for up to ``max_frames`` frames)."""

    def __init__(self, model, device, max_frames, with_vertices, precision=_lib.PRECISION_F16X2):
        self.lib = _lib.load()
        self.ctx = _lib.ctx(device.index)
        self.device, self.max_frames, self.with_vertices = device, int(max_frames), bool(with_vertices)
        g = lambda n: getattr(model, n).detach().to(device=device, dtype=torch.float32).contiguous()
        vt, sd, jr = g("v_template"), g("shapedirs"), g("J_regressor")
        if sd.shape[-1] < 10:
            raise RohmB200Error("body model: shapedirs must hold at least 10 shape components")
        pd = g("posedirs") if with_vertices else None
        lw = g("lbs_weights") if with_vertices else None
        parents = [int(p) for p in getattr(model, "parents").tolist()]
        parents[0] = -1
        if len(parents) != 55 or (with_vertices and tuple(pd.shape) != (486, vt.shape[0] * 3)):
            raise RohmB200Error("body model: expected an SMPL-X layout (55 joints, posedirs [486, V*3])")
        self.V = int(vt.shape[0])
        arr = (C.c_int * 55)(*parents)
        handle = C.c_void_p()
        with torch.cuda.device(device):
            rc = self.lib.rohm_body_create(self.ctx, C.c_void_p(vt.data_ptr()), C.c_void_p(sd.data_ptr()), int(sd.shape[-1]),
                                           C.c_void_p(pd.data_ptr() if pd is not None else 0), C.c_void_p(jr.data_ptr()),
                                           C.c_void_p(lw.data_ptr() if lw is not None else 0), arr, self.V,
                                           self.max_frames, int(with_vertices), precision, C.byref(handle))
        _lib.check(rc, self.ctx)
        self.handle = handle
        # The fused blend + skinning launch writes the vertices with TMA bulk stores when every frame's row starts on a 16-byte
        # boundary: 3 V = 31425 floats does not, so the buffer gets 3 pad floats per frame and the caller a strided [N, V, 3]
        # view of it (same values, `.contiguous()` gives smplx's dense layout).  ROHM_B200_LBS_TMA_STORE=0: dense rows, 4-byte stores.
        self.skin_path = self.lib.rohm_body_skin_path(handle)  # _lib.SKIN_FUSED / SKIN_SPARSE / SKIN_DENSE, -1 without vertices
        self.vertex_pitch = 0
        if self.skin_path == _lib.SKIN_FUSED and os.environ.get("ROHM_B200_LBS_TMA_STORE", "1") != "0":
            pitch = -(-self.V * 3 // 4) * 4
            _lib.check(self.lib.rohm_body_set_vertex_pitch(handle, pitch), self.ctx)
            self.vertex_pitch = pitch

    def _vertex_buffer(self, n):
        if not self.vertex_pitch:
            return torch.empty(n, self.V, 3, device=self.device)
        return torch.empty(n, self.vertex_pitch, device=self.device)[:, :self.V * 3].view(n, self.V, 3)

    def __del__(self):
        h = getattr(self, "handle", None)
        if h:
            try:
                self.lib.rohm_body_destroy(h)
            except Exception:
                pass
            self.handle = None

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def forward(self, global_orient, body_pose, betas, transl, want_vertices, num_joints=55):
        N = global_orient.shape[0]
        f = lambda t, w: t.reshape(N, w).to(device=self.device, dtype=torch.float32).contiguous()
        go, bp, be, tr = f(global_orient, 3), f(body_pose, 63), f(betas, 10), f(transl, 3)
        joints = torch.empty(N, num_joints, 3, device=self.device)
        verts = self._vertex_buffer(N) if want_vertices else None
        rc = self.lib.rohm_body_forward(self.handle, C.c_void_p(go.data_ptr()), C.c_void_p(bp.data_ptr()),
                                        C.c_void_p(be.data_ptr()), C.c_void_p(tr.data_ptr()), N,
                                        C.c_void_p(joints.data_ptr()), num_joints,
                                        C.c_void_p(verts.data_ptr() if verts is not None else 0), self._stream())
        _lib.check(rc, self.ctx)
        return joints, verts

    def from_repr(self, x, mean, std, want_vertices, num_joints=22, channels_last=False, lengths=None):
        """x: normalised [B, 294, 1, T] (or [B, T, 294] with channels_last) -> joints [B, T, num_joints, 3]
        (+ vertices [B, T, V, 3]).  lengths (int32 device [B], see glue.device_lengths): only the clips' own frames are
        computed -> packed joints [sum of lengths, num_joints, 3] (+ vertices [sum of lengths, V, 3]), each frame equal to
        the same frame of the padded call; the sum of lengths, not B * T, has to fit the handle's capacity."""
        if channels_last:
            B, T, _ = x.shape
        else:
            B, _, _, T = x.shape
        clip_off, total = None, 0
        if lengths is not None:
            from .glue import clip_layout
            clip_off, total = clip_layout(lengths, B, T, "from_repr")
        frames = B * T if lengths is None else total
        joints = torch.empty(frames, num_joints, 3, device=self.device)
        verts = self._vertex_buffer(frames) if want_vertices else None
        rc = self.lib.rohm_body_from_repr(self.handle, _p(x), int(bool(channels_last)), _p(mean), _p(std), B, T,
                                          _p(lengths), _p(clip_off), total, _p(joints), num_joints, _p(verts),
                                          self._stream())
        _lib.check(rc, self.ctx)
        if lengths is not None:
            return (joints, verts) if want_vertices else joints
        joints = joints.reshape(B, T, num_joints, 3)
        return (joints, verts.reshape(B, T, self.V, 3)) if want_vertices else joints

    def skating_guidance(self, x0, mean, std, want_loss=False, lengths=None, per_clip=False):
        """lengths: optional int32 device tensor [B] of real frames per clip (None: every clip has T frames).
        per_clip: normalise each clip by its own counts, so clip b's gradient equals the call on clip b alone; the loss
        is then [B, 4] (the four sums per clip) instead of [4].  Its speed sums may differ in the last bits between calls
        (the order of the device's additions); the counts are exact."""
        B, _, _, T = x0.shape
        grad = torch.empty_like(x0)
        loss = (torch.empty(B, 4, device=self.device) if per_clip else torch.empty(4, device=self.device)) if want_loss else None
        rc = self.lib.rohm_skating_guidance(self.handle, _p(x0), _p(mean), _p(std), _p(lengths), B, T, int(bool(per_clip)),
                                            _p(grad), _p(loss), self._stream())
        _lib.check(rc, self.ctx)
        return (grad, loss) if want_loss else grad


    def skating_guidance_global(self, x0, mean, std, reduce_sums):
        """Skating guidance with batch-GLOBAL loss normalisers in a clip-sharded run: this shard's four loss sums are handed
        to ``reduce_sums`` (an in-place all-reduce over the ranks: 4 floats, the one optional intra-step collective of the
        path), then the gradient of this shard is formed with the reduced sums."""
        B, _, _, T = x0.shape
        sums = torch.empty(4, device=self.device)
        rc = self.lib.rohm_skating_guidance_sums(self.handle, C.c_void_p(x0.data_ptr()), C.c_void_p(mean.data_ptr()),
                                                 C.c_void_p(std.data_ptr()), B, T, C.c_void_p(sums.data_ptr()), self._stream())
        _lib.check(rc, self.ctx)
        reduce_sums(sums)
        grad = torch.empty_like(x0)
        rc = self.lib.rohm_skating_guidance_backward(self.handle, C.c_void_p(x0.data_ptr()), C.c_void_p(mean.data_ptr()),
                                                     C.c_void_p(std.data_ptr()), B, T, C.c_void_p(sums.data_ptr()),
                                                     C.c_void_p(grad.data_ptr()), self._stream())
        _lib.check(rc, self.ctx)
        return grad

    def projection_guidance(self, x0, mean, std, cam_affine, focal, center, keypoints_2d, want_loss=False, lengths=None,
                            per_clip=False):
        """d(-loss_2d)/dx0 of guide_2d_projection_with_smpl (reference posenet.py:260-317): x0 [B,294,1,T] normalised,
        cam_affine [B,3,4] canonical -> camera, focal / center [B,2], keypoints_2d [B,>=T,22,3].  per_clip: the mean of
        clip b runs over its own frames, so its gradient equals the call on clip b alone; the loss is then [B] instead of
        [1].  lengths (optional int32 device tensor [B], per_clip only): frames at or past lengths[b] are not read and get
        a zero gradient."""
        B, _, _, T = x0.shape
        if lengths is not None and not per_clip:
            raise RohmB200Error("projection_guidance: lengths need per_clip=True (a batch-wide mean over clips of different "
                                "lengths is not defined)")
        grad = torch.empty_like(x0)
        loss = torch.empty(B if per_clip else 1, device=self.device) if want_loss else None
        rc = self.lib.rohm_projection_guidance(
            self.handle, C.c_void_p(x0.data_ptr()), C.c_void_p(mean.data_ptr()), C.c_void_p(std.data_ptr()), _p(lengths),
            B, T, int(bool(per_clip)), C.c_void_p(cam_affine.data_ptr()), C.c_void_p(focal.data_ptr()),
            C.c_void_p(center.data_ptr()), C.c_void_p(keypoints_2d.data_ptr()), int(keypoints_2d.shape[1]),
            C.c_void_p(grad.data_ptr()), C.c_void_p(loss.data_ptr() if loss is not None else 0), self._stream())
        _lib.check(rc, self.ctx)
        return (grad, loss) if want_loss else grad

    def traj_glue(self, traj_out, repr_clean, traj_mean, traj_std, pose_mean, pose_std, lengths=None):
        """test_amass_full.py:268-311 on the device: -> (composite [B,T,294], traj_full [B,T-1,22]).  lengths: (int32 device
        [B], clip_off int32 device [B+1], their sum) for clips of different lengths, None for clips of T frames."""
        B, T, D = traj_out.shape
        composite = torch.empty(B, T, 294, device=self.device)
        traj_full = torch.empty(B, T - 1, 22, device=self.device)
        lens, clip_off, total = lengths if lengths is not None else (None, None, 0)
        rc = self.lib.rohm_traj_glue(self.handle, _p(traj_out), D, _p(repr_clean), _p(traj_mean), _p(traj_std),
                                     _p(pose_mean), _p(pose_std), B, T, _p(lens), _p(clip_off), total, _p(composite),
                                     _p(traj_full), self._stream())
        _lib.check(rc, self.ctx)
        return composite, traj_full


def kernels_for(model, device, frames, with_vertices):
    """The (cached) BodyKernels of a body-model module -- the package's BodyModel or a real ``smplx`` module (same
    buffer names).  Capacity grows on demand."""
    cache = model.__dict__.setdefault("_rohm_kernels", {})
    key = (str(device), bool(with_vertices))
    k = cache.get(key)
    if k is None or k.max_frames < frames:
        cache[key] = None
        k = BodyKernels(model, torch.device(device), max(int(frames), 1), with_vertices)
        cache[key] = k
    return k


def load_faces(path):
    """The SMPL-X triangles [F,3] (int64) of a model file: ``f`` of ``SMPLX_NEUTRAL.npz``, or of
    ``<path>/smplx/SMPLX_NEUTRAL.npz`` for the directory ``BodyModel.create`` takes.  They are not a ``BodyModel`` buffer,
    so checkpoints keep their state-dict keys."""
    npz = path if os.path.isfile(path) else os.path.join(path, 'smplx', 'SMPLX_NEUTRAL.npz')
    if not os.path.exists(npz):
        raise RohmB200Error(f"load_faces: {npz} not found")
    f = np.asarray(np.load(npz, allow_pickle=True)['f'], dtype=np.int64)
    if f.ndim != 2 or f.shape[1] != 3:
        raise RohmB200Error(f"load_faces: {npz}: 'f' must be [F,3], got {f.shape}")
    return f


class BodyModel(nn.Module):
    NUM_JOINTS = 55
    NUM_BODY_JOINTS = 21

    def __init__(self, tensors):
        super().__init__()
        for name in ("v_template", "shapedirs", "posedirs", "J_regressor", "lbs_weights"):
            self.register_buffer(name, tensors[name].to(torch.float32).contiguous())
        self.register_buffer("parents", torch.tensor(tensors["parents"], dtype=torch.long))
        self._handle = None

    @staticmethod
    def create(body_model_path='', device=None, seed=0, synthetic_ok=None):
        """Loads ``<path>/smplx/SMPLX_NEUTRAL.npz`` (official file layout).  The seeded synthetic SMPL-X-shaped model
        (tests / benchmarks; NOT a human body) is built only on an explicit opt-in: ``body_model_path=''`` (the
        constructor default) or ``synthetic_ok=True``.  A non-empty path without the model file raises -- guiding the
        sampler with a made-up body would be a silent wrong answer."""
        npz = os.path.join(body_model_path or '', 'smplx', 'SMPLX_NEUTRAL.npz')
        if body_model_path and not os.path.exists(npz) and not synthetic_ok:
            raise RohmB200Error(
                f"BodyModel.create: {npz} not found.  Pass the directory that contains smplx/SMPLX_NEUTRAL.npz (the "
                "official SMPL-X download), or body_model_path='' / synthetic_ok=True to opt in to the synthetic "
                "SMPL-X-shaped test model.")
        if body_model_path and os.path.exists(npz):
            d = np.load(npz, allow_pickle=True)
            shapedirs = np.concatenate([d['shapedirs'][:, :, :10], d['shapedirs'][:, :, 300:310]], axis=-1)
            V = d['v_template'].shape[0]
            tensors = {"v_template": torch.from_numpy(np.asarray(d['v_template'], np.float32)),
                       "shapedirs": torch.from_numpy(np.asarray(shapedirs, np.float32)),
                       "posedirs": torch.from_numpy(np.asarray(d['posedirs'], np.float32).reshape(V * 3, -1).T.copy()),
                       "J_regressor": torch.from_numpy(np.asarray(d['J_regressor'], np.float32)),
                       "lbs_weights": torch.from_numpy(np.asarray(d['weights'], np.float32)),
                       "parents": [int(p) for p in np.asarray(d['kintree_table'][0], np.int64)]}
            tensors["parents"][0] = -1
        else:
            tensors = synthetic.smplx_like_model(seed)
        m = BodyModel(tensors)
        return m.to(device) if device is not None else m

    # smplx's own buffer names -> ours, for checkpoints saved from a reference PoseNet (its state dict contains the whole
    # body model under ``smplx_model.*``, reference posenet.py:57)
    def load_smplx_state(self, sd):
        """Adopts the body-model tensors found in a ``smplx_model.*`` state-dict slice (real smplx naming: v_template,
        shapedirs [V,3,10] + expr_dirs [V,3,10], posedirs, J_regressor, lbs_weights, parents); other keys (faces,
        default pose parameters, landmark tables) are not needed by RoHM's calls and are ignored.  Returns the list of
        adopted names."""
        took = []
        if "shapedirs" in sd:
            sdirs = sd["shapedirs"].to(torch.float32)
            if "expr_dirs" in sd and sdirs.shape[-1] == 10:
                sdirs = torch.cat([sdirs, sd["expr_dirs"].to(torch.float32)], dim=-1)
            self.shapedirs = sdirs.to(self.shapedirs.device).contiguous()
            took.append("shapedirs")
        for name in ("v_template", "posedirs", "J_regressor", "lbs_weights"):
            if name in sd:
                setattr(self, name, sd[name].to(device=getattr(self, name).device, dtype=torch.float32).contiguous())
                took.append(name)
        if "parents" in sd:
            par = sd["parents"].to(torch.long).clone()
            par[0] = -1
            self.parents = par.to(self.parents.device)
            took.append("parents")
        self.__dict__.pop("_rohm_kernels", None)
        return took

    def as_dict(self):
        return {"v_template": self.v_template, "shapedirs": self.shapedirs, "posedirs": self.posedirs,
                "J_regressor": self.J_regressor, "lbs_weights": self.lbs_weights, "parents": self.parents.tolist()}

    def _apply(self, fn, *a, **k):
        self.__dict__.pop("_rohm_kernels", None)
        return super()._apply(fn, *a, **k)

    def forward(self, transl=None, global_orient=None, body_pose=None, betas=None, return_verts=True, **zeros):
        """Call-compatible with ``smplx_model(**smplx_params_dict)`` as RoHM uses it
        (motion_representation.py:379-389): jaw / eye / hand poses and expression are accepted and must be zero.
        Returns an object with ``.joints`` [N, 55, 3] and ``.vertices`` [N, V, 3] (a strided view of a 16-byte-pitched buffer
        when the fused launch stores through TMA: same values and shape, ``.contiguous()`` gives smplx's dense layout)."""
        dev = self.v_template.device
        if dev.type != "cuda":
            raise RohmB200Error("BodyModel: the model must live on a CUDA device (no CPU path)")
        for name, val in zeros.items():
            # jaw_pose / leye_pose / reye_pose / left_hand_pose / right_hand_pose / expression: RoHM always passes zeros
            # (motion_representation.py:383-388) and the kernels hard-wire that; anything else must fail loudly.
            if name in ("return_full_pose", "pose2rot", "return_joints"):
                continue
            if isinstance(val, torch.Tensor):
                if val.numel() and bool(torch.count_nonzero(val)):
                    raise RohmB200Error(f"BodyModel.forward: {name} must be all zeros (RoHM's call convention); the "
                                        "CUDA kernels do not evaluate hands / jaw / eyes / expression")
            elif val is not None:
                raise RohmB200Error(f"BodyModel.forward: unsupported argument {name}={val!r}")
        N = global_orient.shape[0]
        k = kernels_for(self, dev, N, with_vertices=return_verts)
        joints, verts = k.forward(global_orient, body_pose, betas, transl, return_verts)
        return BodyOutput(joints=joints, vertices=verts)
