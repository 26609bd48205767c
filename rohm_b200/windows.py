"""Whole recordings in and out of the rounds (SURVEY.md 8f row N4, sliding-window batching).

``encode`` cuts packed recordings into the reference's windows of ``clip_len`` frames (dataloader_video.py:160-183 with
overlap 2, dataloader_amass.py:105-131 with overlap 0), canonicalises each (cano_seq_smplx), encodes its 294-channel
representation (get_repr_smplx) and assembles the batch dicts ``pipeline.run_rounds`` takes, as DataloaderAMASS.__getitem__
builds them without input noise (dataloader_amass.py:319-341).  ``to_recordings`` maps each window's joints back to the
world frame of its recording (the inverse of transf_matrix, eval_prox_egobody.py:177-182).  Both are one kernel launch
(rohm_window_encode / rohm_window_to_world); tensors stay on the GPU.

``encode_video`` builds the batches of the video loader (DataloaderVideo, PROX and EgoBody) from recordings whose
per-frame fits are in each recording's camera frame: the camera instance of the encoder (rohm_window_encode_video), the
keypoints and visibility masks (rohm_window_keypoints) and, for EgoBody, the ground-truth joints in the scene frame
(rohm_window_scene_joints).  Each window's ``cam2world`` rides along in test_batch_pose, so PoseNet's projection guidance
can take a batch of windows of recordings with different cameras.

``encode(..., noise=InputNoise...)`` adds the reference's input noise (dataloader_amass.py:156-227 with sep_noise False,
the paper's setup): noise on each window's canonical SMPL-X parameters (rohm_window_param_noise), FK of the noisy
parameters with the body model, and their representation without re-canonicalisation (rohm_window_encode_canonical).

Only full windows are cut, so a recording shorter than ``clip_len`` gives none, and the frames after a recording's last
window are not covered.  A window's results cover its first clip_len - 2 frames (the PoseNet frames): with overlap 2
consecutive windows tile the recording, with overlap 0 each leaves a 2-frame gap.  ``to_recordings`` reports which frames
a window covers and does not fill the others.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib, glue, noise_streams, ops
from ._lib import RohmB200Error

MAX_CLIP_LEN = 160  # one CTA of one thread per window frame
# channels of the 294-wide row the TrajNet condition keeps with repr_abs_only (dataloader_amass.py:337)
ABS_TRAJ_CHANNELS = (0, 2, 3, 6, 7, 8, 9, 10, 11, 12, 16, 17, 18)
PARAMS = (('global_orient', 3), ('transl', 3), ('betas', 10), ('body_pose', 63))
# a row of Windows.noisy_params: the PARAMS in order, 79 floats
NOISY_ROW = {'global_orient': slice(0, 3), 'transl': slice(3, 6), 'betas': slice(6, 16), 'body_pose': slice(16, 79)}
NOISY_WIDTH = 79
# the reference's order of draws (dataloader_amass.py:159) and each draw's channels per frame
NOISE_DRAWS = (('transl', 3), ('body_pose', 63), ('betas', 10), ('global_orient', 3))
NOISE_SHAPES = {'transl': (3,), 'betas': (10,), 'global_orient': (3,), 'body_pose': (21, 3)}


def window_table(lengths, clip_len=145, overlap=2):
    """[(recording, first frame)] of every window, in order: window k of a recording starts at k * (clip_len - overlap)
    and is cut while it ends inside the recording."""
    stride = clip_len - overlap
    return [(r, s) for r, n in enumerate(lengths) for s in range(0, int(n) - clip_len + 1, stride)]


class Windows:
    """The windows of one ``encode`` call: ``recording`` / ``start`` (int32 device [W]), ``transf`` (world -> canonical
    [W,4,4]), and the recordings' ``lengths`` (ints), ``offsets`` (int32 device [R+1]), ``clip_len`` and ``overlap``.
    With input noise, ``noisy_params`` holds the noisy canonical SMPL-X parameters [W, clip_len, 79] (rows of
    global_orient 3 | transl 3 | betas 10 | body_pose 63 axis-angle, see NOISY_ROW); None without."""

    def __init__(self, recording, start, transf, lengths, offsets, clip_len, overlap, noisy_params=None):
        self.recording, self.start, self.transf = recording, start, transf
        self.lengths, self.offsets, self.clip_len, self.overlap = lengths, offsets, clip_len, overlap
        self.noisy_params = noisy_params

    def __len__(self):
        return int(self.recording.shape[0])


class InputNoise:
    """The input noise of W windows, one entry per window in window order (``window_table``), in the layout and units of
    the reference's preset-noise pickle (smplx_noise_level_*.pkl, one entry per clip): transl [W, clip_len, 3] metres,
    betas [W, clip_len, 10] (per frame), global_orient [W, clip_len, 3] and body_pose [W, clip_len, 21, 3] degrees, added
    to scipy's extrinsic 'zxy' Euler angles of the canonical rotations.  Build it with ``given`` or ``drawn``."""

    def __init__(self, tensors=None, generators=None, stds=None):
        self._tensors, self._generators, self._stds = tensors, generators, stds

    @classmethod
    def given(cls, transl, betas, global_orient, body_pose):
        """Preset noise (load_noise=True): float32 CUDA tensors on one device, shapes as in the class docstring."""
        t = {'transl': transl, 'betas': betas, 'global_orient': global_orient, 'body_pose': body_pose}
        dev = None
        for name, v in t.items():
            if not torch.is_tensor(v):
                raise RohmB200Error(f"InputNoise.given: {name} must be a torch tensor, got {type(v).__name__}")
            if v.device.type != 'cuda':
                raise RohmB200Error(f"InputNoise.given: {name} must be a CUDA tensor, got one on {v.device}")
            if v.dtype != torch.float32:
                raise RohmB200Error(f"InputNoise.given: {name} must be float32, got {v.dtype}")
            if dev is not None and v.device != dev:
                raise RohmB200Error(f"InputNoise.given: {name} lives on {v.device}, transl on {dev}")
            dev = v.device
            want = 2 + len(NOISE_SHAPES[name])
            if v.dim() != want or tuple(v.shape[2:]) != NOISE_SHAPES[name]:
                raise RohmB200Error(f"InputNoise.given: {name} must be [W, clip_len, {', '.join(map(str, NOISE_SHAPES[name]))}]"
                                    f", got {tuple(v.shape)}")
            if tuple(v.shape[:2]) != tuple(transl.shape[:2]):
                raise RohmB200Error(f"InputNoise.given: {name} covers [W, clip_len] = {tuple(v.shape[:2])}, transl "
                                    f"{tuple(transl.shape[:2])}")
        return cls(tensors={k: v.contiguous() for k, v in t.items()})

    @classmethod
    def drawn(cls, generators, std_global_rot=3.0, std_body_rot=3.0, std_transl=0.03, std_betas=0.1):
        """Noise drawn on the device from one CUDA torch.Generator per window (defaults: test_amass_full.py's noise level
        3).  Window w gets exactly ``std * torch.randn(shape, generator=generators[w])`` for each parameter, in the
        reference's order (transl [clip_len, 3], body_pose [clip_len*21, 3], betas [clip_len, 10], global_orient
        [clip_len, 3]), and each generator's offset advances as those four torch draws would advance it.  The draws
        happen in ``encode``, after its checks."""
        if not isinstance(generators, (list, tuple)):
            raise RohmB200Error(f"InputNoise.drawn: generators must be a list or tuple of torch.Generator, got "
                                f"{type(generators).__name__}")
        stds = {'global_orient': std_global_rot, 'body_pose': std_body_rot, 'transl': std_transl, 'betas': std_betas}
        for name, v in stds.items():
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not np.isfinite(v) or v < 0:
                raise RohmB200Error(f"InputNoise.drawn: the standard deviation of {name} must be a finite number >= 0, "
                                    f"got {v!r}")
        return cls(generators=list(generators), stds={k: float(v) for k, v in stds.items()})

    def _check(self, W, clip_len, dev):
        """Refuses a noise that does not fit W windows of clip_len frames on `dev`, before anything runs."""
        if W == 0:
            raise RohmB200Error("windows.encode: input noise for a batch that cuts no window (every recording is shorter "
                                "than clip_len)")
        if self._tensors is not None:
            got = tuple(self._tensors['transl'].shape[:2])
            if got != (W, clip_len):
                raise RohmB200Error(f"windows.encode: the input noise covers [W, clip_len] = {got}, the recordings cut "
                                    f"{W} windows of {clip_len} frames")
            if self._tensors['transl'].device != dev:
                raise RohmB200Error(f"windows.encode: the input noise lives on {self._tensors['transl'].device}, the "
                                    f"parameters on {dev}")
            return
        gens = self._generators
        if len(gens) != W:
            raise RohmB200Error(f"windows.encode: InputNoise.drawn holds {len(gens)} generators, the recordings cut {W} "
                                "windows; give every window its own")
        if len({id(g) for g in gens}) != len(gens):
            raise RohmB200Error("InputNoise.drawn: the same generator object appears twice; give every window its own")
        step = noise_streams.MAX_CLIPS
        for i in range(0, W, step):
            try:
                noise_streams.check_generators({'generators': gens[i:i + step]}, len(gens[i:i + step]), dev)
            except RohmB200Error as e:
                raise RohmB200Error(f"InputNoise.drawn (windows {i}..): {e}") from None

    def _tensors_for(self, clip_len, dev):
        """The noise tensors: the given ones, or the draws (at most MAX_CLIPS generators per launch; every generator's
        draws are its own, so the chunking changes no bit)."""
        if self._tensors is not None:
            return self._tensors
        W = len(self._generators)
        out = {}
        for name, width in NOISE_DRAWS:
            t = torch.empty(W, clip_len, width, device=dev)
            for i in range(0, W, noise_streams.MAX_CLIPS):
                chunk = self._generators[i:i + noise_streams.MAX_CLIPS]
                streams = noise_streams.NoiseStreams(chunk, dev)
                t[i:i + len(chunk)] = ops.randn_clips(streams, [len(chunk), clip_len, width], True)
                streams.close()
            out[name] = t.mul_(self._stds[name]).reshape(W, clip_len, *NOISE_SHAPES[name])
        return out


def _check_shape(clip_len, overlap):
    if not 3 <= clip_len <= MAX_CLIP_LEN or not 0 <= overlap <= 2:
        raise RohmB200Error(f"windows: clip_len={clip_len}, overlap={overlap}; windows of 3 to {MAX_CLIP_LEN} frames with an "
                            "overlap of 0 to 2 frames (so that no recording frame lies in two windows' pose frames)")


def encode(body_model, params, lengths, pose_dataset, traj_dataset, clip_len=145, overlap=2, noise=None):
    """params: SMPL-X parameters of R recordings packed frame after frame (CUDA tensors global_orient [N,3], transl [N,3],
    betas [N,10], body_pose [N,63] axis-angle, N = sum of lengths, z up); lengths: frames per recording (ints).  World joints
    come from ``body_model`` (FK only).  Returns (test_batch_traj, test_batch_pose, windows):

    * test_batch_traj: motion_repr_clean / motion_repr_noisy [W, clip_len-1, 294] z-scored with traj_dataset's statistics,
      cond [W, clip_len-1, 13] (the repr_abs_only channels; the first traj_feat_dim channels otherwise) and control_cond
      [W, clip_len-1, pose_feat_dim];
    * test_batch_pose: motion_repr_clean / motion_repr_noisy z-scored with pose_dataset's statistics;
    * windows: the window table and transf (``Windows``), for ``to_recordings``.

    Each window's rows depend on its own frames only: the same in any batch, order or packing of recordings.

    noise: an ``InputNoise`` for the W windows, or None (motion_repr_noisy is then a copy of motion_repr_clean).  With
    noise, the dicts are the ones DataloaderAMASS.__getitem__ builds with input_noise (dataloader_amass.py:317-341):
    motion_repr_noisy is the representation of the noisy window, in test_batch_pose with its first
    pose_dataset.traj_feat_dim channels replaced by the clean ones; test_batch_traj's cond is the noisy trajectory and
    control_cond the clean local pose; both dicts get noisy_joints [W, clip_len, 22, 3] (canonical, from FK of the noisy
    parameters with ``body_model``), and windows.noisy_params the noisy parameters.  One deliberate difference: with
    load_noise=False the reference's pose and traj datasets each draw their own noise from numpy's global stream; here
    one noise per window feeds both dicts, as the reference's default load_noise=True does.  Each window's noisy rows
    depend on its own frames and its own noise only."""
    _check_noise_type(noise)
    p, lengths = _packed_params(params, lengths, clip_len, overlap)
    W = len(window_table(lengths, clip_len, overlap))
    _check_noise(noise, W, clip_len, p['transl'].device)
    joints = None
    if W:
        joints = body_model(transl=p['transl'], global_orient=p['global_orient'], body_pose=p['body_pose'],
                            betas=p['betas'], return_verts=False).joints[:, 0:22].contiguous()
    return _encode(p, joints, lengths, pose_dataset, traj_dataset, clip_len, overlap, noise, body_model)


def encode_joints(params, joints, lengths, pose_dataset, traj_dataset, clip_len=145, overlap=2, noise=None,
                  body_model=None):
    """``encode`` with the recordings' 22-joint world positions given (joints [N,22,3], packed like params), as the
    reference loaders read them from preprocessed files.  With ``noise``, ``body_model`` gives the noisy joints by FK, as
    the AMASS loader does (dataloader_amass.py:194-206)."""
    _check_noise_type(noise)
    if noise is not None and body_model is None:
        raise RohmB200Error("windows.encode_joints: input noise needs body_model, which gives the noisy joints by FK")
    p, lengths = _packed_params(params, lengths, clip_len, overlap)
    joints = glue._f32c(joints, "windows.encode_joints: joints")
    if joints.numel() != sum(lengths) * 66:
        raise RohmB200Error(f"windows.encode_joints: joints must hold [{sum(lengths)}, 22, 3], got {tuple(joints.shape)}")
    _check_noise(noise, len(window_table(lengths, clip_len, overlap)), clip_len, p['transl'].device)
    return _encode(p, joints, lengths, pose_dataset, traj_dataset, clip_len, overlap, noise, body_model)


def _check_noise_type(noise):
    if noise is not None and not isinstance(noise, InputNoise):
        raise RohmB200Error(f"windows.encode: noise must be an InputNoise (InputNoise.given / .drawn) or None, got "
                            f"{type(noise).__name__}")


def _check_noise(noise, W, clip_len, dev):
    if noise is not None:
        noise._check(W, clip_len, dev)


def _packed_params(params, lengths, clip_len, overlap):
    _check_shape(clip_len, overlap)
    lengths = tuple(int(n) for n in lengths)
    if not lengths or min(lengths) < 0:
        raise RohmB200Error(f"windows.encode: lengths must be one frame count >= 0 per recording, got {lengths}")
    total = sum(lengths)
    p = {}
    for name, width in PARAMS:
        t = glue._f32c(params[name], f"windows.encode: params['{name}']")
        if t.numel() != total * width:
            raise RohmB200Error(f"windows.encode: params['{name}'] must hold [{total}, {width}] (the packed recordings), got "
                                f"{tuple(t.shape)}")
        p[name] = t.reshape(total, width)
    return p, lengths


def _encode(p, joints, lengths, pose_dataset, traj_dataset, clip_len, overlap, noise=None, body_model=None):
    dev = p['transl'].device
    tm, ts = glue.stats_on(traj_dataset, dev)
    pm, ps = glue.stats_on(pose_dataset, dev)
    if any(t.numel() != glue.BODY_FEAT_DIM for t in (tm, ts, pm, ps)):
        raise RohmB200Error("windows.encode: the datasets' Mean / Std must have 294 entries")
    W, T1 = len(window_table(lengths, clip_len, overlap)), clip_len - 1
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    offsets = torch.from_numpy(off).to(dev)
    rec = torch.empty(W, dtype=torch.int32, device=dev)
    start = torch.empty(W, dtype=torch.int32, device=dev)
    transf = torch.empty(W, 4, 4, device=dev)
    rt = torch.empty(W, T1, glue.BODY_FEAT_DIM, device=dev)
    rp = torch.empty(W, T1, glue.BODY_FEAT_DIM, device=dev)
    if W > 0:
        lib, ctx = _lib.load(), _lib.ctx(dev.index)
        n = C.c_int(0)
        rc = lib.rohm_window_encode(ctx, glue._p(p['global_orient']), glue._p(p['transl']), glue._p(p['betas']),
                                    glue._p(p['body_pose']), glue._p(joints), (C.c_int * len(off))(*off.tolist()),
                                    glue._p(offsets), len(lengths), clip_len, overlap, glue._p(tm), glue._p(ts),
                                    glue._p(pm), glue._p(ps), W, C.byref(n), glue._p(rec), glue._p(start), glue._p(transf),
                                    glue._p(rt), glue._p(rp), glue._stream(dev))
        _lib.check(rc, ctx)
        if n.value != W:
            raise RohmB200Error(f"windows.encode: the library cut {n.value} windows, the window rule {W}")
    tfd, pfd = traj_dataset.traj_feat_dim, traj_dataset.pose_feat_dim
    win = Windows(rec, start, transf, lengths, offsets, clip_len, overlap)
    if noise is None:
        cond = rt[..., list(ABS_TRAJ_CHANNELS)] if tfd == len(ABS_TRAJ_CHANNELS) else rt[..., 0:tfd].clone()
        test_batch_traj = {'motion_repr_clean': rt, 'motion_repr_noisy': rt.clone(), 'cond': cond,
                           'control_cond': rt[..., -pfd:].contiguous()}
        test_batch_pose = {'motion_repr_clean': rp, 'motion_repr_noisy': rp.clone()}
        return test_batch_traj, test_batch_pose, win

    # dataloader_amass.py:156-215: noisy canonical parameters, their FK, their representation (not re-canonicalised)
    n = noise._tensors_for(clip_len, dev)
    lib, ctx = _lib.load(), _lib.ctx(dev.index)
    noisy = torch.empty(W * clip_len, NOISY_WIDTH, device=dev)
    rc = lib.rohm_window_param_noise(ctx, glue._p(p['global_orient']), glue._p(p['transl']), glue._p(p['betas']),
                                     glue._p(p['body_pose']), glue._p(joints), glue._p(offsets), glue._p(rec),
                                     glue._p(start), glue._p(transf), W, clip_len, glue._p(n['transl']),
                                     glue._p(n['betas']), glue._p(n['global_orient']), glue._p(n['body_pose']),
                                     glue._p(noisy), glue._stream(dev))
    _lib.check(rc, ctx)
    nj = body_model(**{k: noisy[:, s] for k, s in NOISY_ROW.items()}, return_verts=False).joints[:, 0:22].contiguous()
    nt = torch.empty(W, T1, glue.BODY_FEAT_DIM, device=dev)
    npose = torch.empty(W, T1, glue.BODY_FEAT_DIM, device=dev)
    rc = lib.rohm_window_encode_canonical(ctx, glue._p(noisy), glue._p(nj), W, clip_len, glue._p(tm), glue._p(ts),
                                          glue._p(pm), glue._p(ps), glue._p(nt), glue._p(npose), glue._stream(dev))
    _lib.check(rc, ctx)
    # __getitem__ (:317-341): PoseNet is conditioned on the clean trajectory (task 'pose'); TrajNet on the noisy trajectory
    # with the clean local pose as its control signal (task 'traj')
    npose[..., 0:pose_dataset.traj_feat_dim] = rp[..., 0:pose_dataset.traj_feat_dim]
    noisy_joints = nj.reshape(W, clip_len, 22, 3)
    cond = nt[..., list(ABS_TRAJ_CHANNELS)] if tfd == len(ABS_TRAJ_CHANNELS) else nt[..., 0:tfd].clone()
    test_batch_traj = {'motion_repr_clean': rt, 'motion_repr_noisy': nt, 'cond': cond,
                       'control_cond': rt[..., -pfd:].contiguous(), 'noisy_joints': noisy_joints}
    test_batch_pose = {'motion_repr_clean': rp, 'motion_repr_noisy': npose, 'noisy_joints': noisy_joints.clone()}
    win.noisy_params = noisy.reshape(W, clip_len, NOISY_WIDTH)
    return test_batch_traj, test_batch_pose, win


VIDEO_DATASETS = ('prox', 'egobody')
DIST_LENGTHS = (4, 5, 8)  # OpenCV distortion vectors the video loaders' Color.json carry: k1 k2 p1 p2 [k3 [k4 k5 k6]]
# Q = Rx(+90 deg): (x, y, z) -> (x, -z, y), EgoBody's y-up scene frame to the z-up frame cano_seq_smplx takes (DESIGN §4.14)
Y_UP_TO_Z_UP = np.array([[1.0, 0.0, 0.0], [0.0, 0.0, -1.0], [0.0, 1.0, 0.0]])


def _host64(v, name, shape):
    """A small per-recording array as finite float64 numpy of `shape` (None entries: any size), refused otherwise."""
    a = v.detach().cpu().double().numpy() if torch.is_tensor(v) else np.asarray(v, dtype=np.float64)
    if a.ndim != len(shape) or any(w is not None and a.shape[i] != w for i, w in enumerate(shape)):
        want = ", ".join("n" if w is None else str(w) for w in shape)
        raise RohmB200Error(f"windows.encode_video: {name} must be [{want}], got {tuple(a.shape)}")
    if not np.isfinite(a).all():
        raise RohmB200Error(f"windows.encode_video: {name} holds a non-finite value")
    return a


def encode_video(body_model, params, lengths, dataset, cam2world, focal_length, camera_center, camera_mtx, dist,
                 keypoints, depth_mask, pose_dataset, traj_dataset, floor=None, clip_len=145, overlap=2,
                 keypoints_float64=None, gt_params=None, gt_body_model=None, master2world=None, noise=None):
    """The batches of the reference's DataloaderVideo (dataloader_video.py) for R recordings packed frame after frame.

    params: the initial SMPL-X fits in each recording's camera frame, as the per-frame 000.pkl holds them (CUDA tensors
    global_orient [N,3], transl [N,3], betas [N,10], body_pose [N,63]); lengths: frames per recording; dataset: 'prox'
    (z-up scene) or 'egobody' (y-up scene).  Per recording (tensors or arrays, any device): cam2world [R,4,4] (for an
    EgoBody sub view, master2world @ trans_subtomain as the loader composes it), the colour camera focal_length [R,2],
    camera_center [R,2], camera_mtx [R,3,3] and dist [R,n], n in (4, 5, 8), and floor [R] (None: every window takes its
    own minimum; a preset height, where 0.0 also takes the window minimum, as the reference's ``if
    preset_floor_height:`` does).  Per frame (CUDA): keypoints [N,25,3] (OpenPose BODY_25 from the json, zeros where no
    person was found) and depth_mask [N,25] (mask_joint.npy).  keypoints_float64 [R] bools: the recording's keypoint
    array is float64 in the loader (a frame had no person, np.zeros is float64), which sets the precision of conf > 0.2;
    None derives it from the frames whose keypoints are all zero.  For EgoBody with ground truth: gt_params (fits in the
    master camera frame, packed like params), gt_body_model and master2world [R,4,4].

    Returns (test_batch_traj, test_batch_pose, windows): every key DataloaderVideo.__getitem__ emits for task 'traj' and
    'pose' as CUDA float32 tensors with a leading W, except frame_name (host strings: windows.recording / start index the
    caller's own name lists); test_batch_pose also carries cam2world [W,4,4], the camera of each window's recording, which
    PoseNet's projection guidance uses in place of dataset.cam_R / cam_t.  windows.transf is the reference's scene ->
    canonical transf_matrix, so ``to_recordings`` returns scene coordinates (y up for EgoBody).  The video loader adds no
    input noise: passing ``noise`` is refused."""
    if noise is not None:
        raise RohmB200Error("windows.encode_video: the video loader adds no input noise; noise must be None")
    if dataset not in VIDEO_DATASETS:
        raise RohmB200Error(f"windows.encode_video: dataset must be one of {VIDEO_DATASETS}, got {dataset!r}")
    _check_shape(clip_len, overlap)
    lengths = tuple(int(n) for n in lengths)
    if not lengths or min(lengths) < 0:
        raise RohmB200Error(f"windows.encode_video: lengths must be one frame count >= 0 per recording, got {lengths}")
    R, N = len(lengths), sum(lengths)
    c2w = _host64(cam2world, "cam2world", (R, 4, 4))
    f = _host64(focal_length, "focal_length", (R, 2))
    c = _host64(camera_center, "camera_center", (R, 2))
    K = _host64(camera_mtx, "camera_mtx", (R, 3, 3))
    k = _host64(dist, "dist", (R, None))
    if k.shape[1] not in DIST_LENGTHS:
        raise RohmB200Error(f"windows.encode_video: dist must hold {DIST_LENGTHS} coefficients per recording, got "
                            f"{k.shape[1]}")
    fl = np.zeros(R) if floor is None else _host64(floor, "floor", (R,))
    for name, t, shape in (("keypoints", keypoints, (N, 25, 3)), ("depth_mask", depth_mask, (N, 25))):
        if not hasattr(t, "shape") or tuple(t.shape) != shape:
            raise RohmB200Error(f"windows.encode_video: {name} must be {list(shape)}, got "
                                f"{tuple(getattr(t, 'shape', ()))}")
    if keypoints_float64 is not None and len(keypoints_float64) != R:
        raise RohmB200Error(f"windows.encode_video: keypoints_float64 must hold one flag per recording ({R}), got "
                            f"{len(keypoints_float64)}")
    with_gt = gt_params is not None
    if with_gt != (gt_body_model is not None) or with_gt != (master2world is not None):
        raise RohmB200Error("windows.encode_video: the ground truth needs gt_params, gt_body_model and master2world "
                            "together")
    if with_gt and dataset != 'egobody':
        raise RohmB200Error("windows.encode_video: ground-truth fits are an EgoBody input")
    m2w = _host64(master2world, "master2world", (R, 4, 4)) if with_gt else None
    p, _ = _packed_params(params, lengths, clip_len, overlap)
    dev = p['transl'].device
    kp = glue._f32c(keypoints, "windows.encode_video: keypoints")
    dm = glue._f32c(depth_mask, "windows.encode_video: depth_mask")
    gp = _packed_params(gt_params, lengths, clip_len, overlap)[0] if with_gt else None
    for name, t in (("keypoints", kp), ("depth_mask", dm)) + ((("gt_params", gp['transl']),) if with_gt else ()):
        if t.device != dev:
            raise RohmB200Error(f"windows.encode_video: {name} lives on {t.device}, the parameters on {dev}")
    tm, ts = glue.stats_on(traj_dataset, dev)
    pm, ps = glue.stats_on(pose_dataset, dev)
    if any(t.numel() != glue.BODY_FEAT_DIM for t in (tm, ts, pm, ps)):
        raise RohmB200Error("windows.encode_video: the datasets' Mean / Std must have 294 entries")

    # the recording's camera -> z-up scene map, in float32 as the loader applies cam2world.float(); for EgoBody Q is a
    # permutation with one sign, so Q A is exact
    c2w32 = c2w.astype(np.float32)
    A = c2w32[:, 0:3, :]
    if dataset == 'egobody':
        A = np.stack([A[:, 0], -A[:, 2], A[:, 1]], axis=1)
    cam = torch.from_numpy(np.ascontiguousarray(A.reshape(R, 12))).to(dev)
    floors = torch.from_numpy(fl.astype(np.float32)).to(dev)
    W, L, T1 = len(window_table(lengths, clip_len, overlap)), clip_len, clip_len - 1
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)
    offsets = torch.from_numpy(off).to(dev)
    rec = torch.empty(W, dtype=torch.int32, device=dev)
    start = torch.empty(W, dtype=torch.int32, device=dev)
    transf = torch.empty(W, 4, 4, device=dev)
    rt = torch.empty(W, T1, glue.BODY_FEAT_DIM, device=dev)
    rp = torch.empty(W, T1, glue.BODY_FEAT_DIM, device=dev)
    cano_joints = torch.empty(W, L, 22, 3, device=dev)
    scene_joints = torch.empty(W, L, 22, 3, device=dev)
    cano_params = torch.empty(W, L, NOISY_WIDTH, device=dev)
    kp_out = torch.empty(W, L, 22, 3, device=dev)
    vis = torch.empty(W, L, 22, device=dev)
    vec = torch.empty(W, L, glue.BODY_FEAT_DIM, device=dev)
    gt_scene = torch.empty(W, L, 22, 3, device=dev) if with_gt else None
    if W > 0:
        lib, ctx = _lib.load(), _lib.ctx(dev.index)
        joints = body_model(transl=p['transl'], global_orient=p['global_orient'], body_pose=p['body_pose'],
                            betas=p['betas'], return_verts=False).joints[:, 0:22].contiguous()
        n = C.c_int(0)
        rc = lib.rohm_window_encode_video(ctx, glue._p(p['global_orient']), glue._p(p['transl']), glue._p(p['betas']),
                                          glue._p(p['body_pose']), glue._p(joints), (C.c_int * len(off))(*off.tolist()),
                                          glue._p(offsets), R, clip_len, overlap, glue._p(cam), glue._p(floors),
                                          int(dataset == 'egobody'), glue._p(tm), glue._p(ts), glue._p(pm), glue._p(ps),
                                          W, C.byref(n), glue._p(rec), glue._p(start), glue._p(transf), glue._p(rt),
                                          glue._p(rp), glue._p(cano_joints), glue._p(scene_joints),
                                          glue._p(cano_params), glue._stream(dev))
        _lib.check(rc, ctx)
        if n.value != W:
            raise RohmB200Error(f"windows.encode_video: the library cut {n.value} windows, the window rule {W}")
        if keypoints_float64 is None:
            empty = (kp.reshape(N, 75) == 0).all(dim=1).cpu().numpy()
            conf64 = torch.tensor([int(empty[off[r]:off[r + 1]].any()) for r in range(R)], dtype=torch.uint8, device=dev)
        else:
            conf64 = torch.tensor([1 if b else 0 for b in keypoints_float64], dtype=torch.uint8, device=dev)
        kpad = np.zeros((R, 14))
        kpad[:, :k.shape[1]] = k
        Kd = torch.from_numpy(np.ascontiguousarray(K.reshape(R, 9))).to(dev)
        kd = torch.from_numpy(kpad).to(dev)
        rc = lib.rohm_window_keypoints(ctx, glue._p(kp), glue._p(dm), glue._p(conf64), glue._p(Kd), glue._p(kd),
                                       int(dataset == 'prox'), glue._p(offsets), glue._p(rec), glue._p(start), W, L,
                                       glue._p(kp_out), glue._p(vis), glue._p(vec), glue._stream(dev))
        _lib.check(rc, ctx)
        if with_gt:
            gj = gt_body_model(transl=gp['transl'], global_orient=gp['global_orient'], body_pose=gp['body_pose'],
                               betas=gp['betas'], return_verts=False).joints[:, 0:22].contiguous()
            mcam = torch.from_numpy(np.ascontiguousarray(m2w.astype(np.float32)[:, 0:3, :].reshape(R, 12))).to(dev)
            rc = lib.rohm_window_scene_joints(ctx, glue._p(gj), glue._p(mcam), glue._p(offsets), glue._p(rec),
                                              glue._p(start), W, L, glue._p(gt_scene), glue._stream(dev))
            _lib.check(rc, ctx)
    ri = rec.long()
    per_rec = lambda a: torch.from_numpy(np.ascontiguousarray(a.astype(np.float32))).to(dev)[ri]
    common = {'noisy_joints': cano_joints, 'noisy_joints_scene_coord': scene_joints, 'transf_matrix': transf,
              'cano_smplx_params_dict': {k_: cano_params[..., s_].contiguous() for k_, s_ in NOISY_ROW.items()},
              'focal_length': per_rec(f), 'camera_center': per_rec(c), 'keypoints_2d': kp_out,
              'mask_joint_vis': vis, 'mask_vec_vis': vec}
    if with_gt:
        common['gt_joints_scene_coord'] = gt_scene
    tfd, pfd = traj_dataset.traj_feat_dim, traj_dataset.pose_feat_dim
    cond = rt[..., list(ABS_TRAJ_CHANNELS)] if tfd == len(ABS_TRAJ_CHANNELS) else rt[..., 0:tfd].clone()
    test_batch_traj = dict(common, motion_repr_noisy=rt, cond=cond, control_cond=rt[..., -pfd:].contiguous())
    test_batch_pose = {key: ({a: b.clone() for a, b in v.items()} if isinstance(v, dict) else v.clone())
                       for key, v in common.items()}
    test_batch_pose.update(motion_repr_noisy=rp, cam2world=per_rec(c2w))
    return test_batch_traj, test_batch_pose, Windows(rec, start, transf, lengths, offsets, clip_len, overlap)


def to_recordings(windows, joints):
    """joints: each window's clip_len - 2 pose frames in its canonical frame, [W, clip_len-2, 22, 3] or packed
    [W*(clip_len-2), 22, 3] (e.g. reconstruct_outputs' rec_ric_data_rec_from_smpl) -> (world, covered): per recording
    world-frame joints [lengths[r], 22, 3] and a bool mask [lengths[r]] of the frames a window covers.  Frames no window
    covers are zero."""
    W, P = len(windows), windows.clip_len - 2
    dev = windows.offsets.device
    j = glue._f32c(joints, "windows.to_recordings: joints")
    if j.numel() != W * P * 22 * 3:
        raise RohmB200Error(f"windows.to_recordings: joints must hold [{W} * {P}, 22, 3] (pose frames of every window), got "
                            f"{tuple(j.shape)}")
    total = sum(windows.lengths)
    world = torch.empty(total, 22, 3, device=dev)
    covered = torch.empty(total, dtype=torch.uint8, device=dev)
    if total > 0:
        lib, ctx = _lib.load(), _lib.ctx(dev.index)
        rc = lib.rohm_window_to_world(ctx, glue._p(j), glue._p(windows.recording), glue._p(windows.start),
                                      glue._p(windows.transf), W, windows.clip_len, glue._p(windows.offsets), total,
                                      glue._p(world), glue._p(covered), glue._stream(dev))
        _lib.check(rc, ctx)
    n = list(windows.lengths)
    return list(torch.split(world, n)), list(torch.split(covered.bool(), n))
