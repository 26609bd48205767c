"""ctypes binding of the C-ABI library (include/rohm_b200.h -> rohm_b200/librohm_b200.so).

The product path has no CPU fallback: if the library is missing or no sm_90 (H100) device is present, every entry point
raises ``RohmB200Error`` with the reason.  Importing this module never touches the GPU; the library is loaded on
first use.
"""
import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "librohm_b200.so")

ROHM_OK = 0
PRECISION_TF32X3 = 3
PRECISION_F16X2 = 2
PRECISION_TF32 = 1
SKIN_FUSED, SKIN_SPARSE, SKIN_DENSE = 0, 1, 2  # rohm_body_skin_path
DDPM_COEFS = 8


class RohmB200Error(RuntimeError):
    pass


class PoseNetLayerW(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "in_proj_w", "in_proj_b", "out_proj_w", "out_proj_b", "lin1_w", "lin1_b", "lin2_w", "lin2_b",
        "norm1_w", "norm1_b", "norm2_w", "norm2_b")]


class PoseNetW(C.Structure):
    _fields_ = [("d_model", C.c_int), ("ff_size", C.c_int), ("num_layers", C.c_int), ("num_heads", C.c_int),
                ("in_feats", C.c_int), ("out_feats", C.c_int), ("traj_feats", C.c_int), ("pe_len", C.c_int)] + \
               [(n, C.c_void_p) for n in ("in_w", "in_b", "cond_w", "cond_b", "pe", "t0_w", "t0_b", "t2_w", "t2_b",
                                          "out_w", "out_b")] + [("layers", C.POINTER(PoseNetLayerW))]


# name -> (restype, argtypes).  Kept in one table so tests can check it against the header.
_p, _i, _i64, _f = C.c_void_p, C.c_int, C.c_int64, C.c_float
SIGNATURES = {
    "rohm_version": (_i, []),
    "rohm_ctx_create": (_i, [_i, C.POINTER(_p)]),
    "rohm_ctx_destroy": (None, [_p]),
    "rohm_last_error": (C.c_char_p, [_p]),
    "rohm_ddpm_step": (_i, [_p, _p, _p, _p, _p, _p, _i, _p, _i64, _i64, _p, _i64, _p]),
    "rohm_ddpm_step_philox": (_i, [_p, _p, _p, _p, _p, _i, _p, _i64, _i64, _p, _i64, C.c_uint64, C.c_uint64,
                                    C.POINTER(C.c_uint64), _p]),
    "rohm_randn_clips": (_i, [_p, _p, _i, _i, _i, _i, C.POINTER(_i), _p, C.c_uint64, C.POINTER(C.c_uint64), _p]),
    "rohm_ddpm_step_philox_clips": (_i, [_p, _p, _p, _p, _p, _i, _p, _i, _i, _i, _i, C.POINTER(_i), _p, _i64, _p,
                                          C.c_uint64, C.POINTER(C.c_uint64), _p]),
    "rohm_q_sample": (_i, [_p, _p, _p, _p, _i64, _f, _f, _p]),
    "rohm_ddim_step": (_i, [_p, _p, _p, _p, _p, _i64, _f, _f, _f, _f, _f, _p]),
    "rohm_posenet_create": (_i, [_p, C.POINTER(PoseNetW), _i, _i, _i, C.POINTER(_p)]),
    "rohm_posenet_destroy": (None, [_p]),
    "rohm_posenet_set_cond": (_i, [_p, _p, _i, _i, _p]),
    "rohm_posenet_set_lengths": (_i, [_p, C.POINTER(_i), _i]),
    "rohm_posenet_forward": (_i, [_p, _p, _p, _p, _i, _i, _p]),
    "rohm_posenet_sample_step": (_i, [_p, _p, _p, _p, _p, _p, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), _i, _i, _p]),
    "rohm_posenet_sample_step_clips": (_i, [_p, _p, _p, _p, _p, _p, _p, C.c_uint64, C.POINTER(C.c_uint64), _i, _i, _p]),
    "rohm_posenet_profile":(_i, [_p, _p, _p, _p, _i, _i, _p, C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    "rohm_posenet_set_option": (_i, [_p, _i, _i]),
    "rohm_posenet_launches_per_forward": (_i, [_p]),
    "rohm_trajnet_create": (_i, [_p, _i, C.POINTER(C.c_char_p), C.POINTER(_p), C.POINTER(_i64), _i, _i, _i, _i, _i, _i,
                                 _i, _i, _i, C.POINTER(_p)]),
    "rohm_trajnet_create_batch_invariant": (_i, [_p, _i, C.POINTER(C.c_char_p), C.POINTER(_p), C.POINTER(_i64), _i, _i,
                                                 _i, _i, _i, _i, _i, _i, _i, C.POINTER(_p)]),
    "rohm_trajnet_destroy": (None, [_p]),
    "rohm_trajnet_set_cond": (_i, [_p, _p, _p, _i, _p]),
    "rohm_trajnet_set_lengths": (_i, [_p, C.POINTER(_i), _i]),
    "rohm_trajnet_forward": (_i, [_p, _p, _p, _p, _i, _p]),
    "rohm_trajnet_sample_step": (_i, [_p, _p, _p, _p, _p, _p, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), _i, _p]),
    "rohm_trajnet_sample_step_clips": (_i, [_p, _p, _p, _p, _p, _p, _p, C.c_uint64, C.POINTER(C.c_uint64), _i, _p]),
    "rohm_trajnet_set_option":(_i, [_p, _i, _i]),
    "rohm_trajnet_launches_per_forward": (_i, [_p]),
    "rohm_body_create": (_i, [_p, _p, _p, _i, _p, _p, _p, C.POINTER(C.c_int), _i, _i64, _i, _i, C.POINTER(_p)]),
    "rohm_body_destroy": (None, [_p]),
    "rohm_body_skin_path": (_i, [_p]),
    "rohm_body_set_vertex_pitch": (_i, [_p, _i64]),
    "rohm_body_forward": (_i, [_p, _p, _p, _p, _p, _i64, _p, _i, _p, _p]),
    "rohm_body_from_repr": (_i, [_p, _p, _i, _p, _p, _i, _i, _p, _p, _i64, _p, _i, _p, _p]),
    "rohm_skating_guidance": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _p, _p, _p]),
    "rohm_skating_guidance_sums": (_i, [_p, _p, _p, _p, _i, _i, _p, _p]),
    "rohm_skating_guidance_backward": (_i, [_p, _p, _p, _p, _i, _i, _p, _p, _p]),
    "rohm_projection_guidance": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _p, _p, _p, _p, _i, _p, _p, _p]),
    "rohm_traj_glue": (_i, [_p, _p, _i, _p, _p, _p, _p, _p, _i, _i, _p, _p, _i64, _p, _p, _p]),
    "rohm_traj_repr_from_joints": (_i, [_p, _p, _p, _p, _p, _p, _i, _i, _p, _p, _p, _p]),
    "rohm_pose_to_control_cond": (_i, [_p, _p, _i, _i, _i, _i, _i, _p, _p, _p]),
    "rohm_build_pose_cond": (_i, [_p, _p, _i, _i, _p, _p, _p, _p, _i, _i, _i, _p, _p, _i, _p, _p]),
    "rohm_rot6d_to_aa": (_i, [_p, _p, _i64, _p, _p, _p]),
    "rohm_joints_from_traj": (_i, [_p, _p, _i, _p, _p, _i, _i, _p, _p, _i64, _i, _p, _p]),
    "rohm_window_encode": (_i, [_p, _p, _p, _p, _p, _p, C.POINTER(_i), _p, _i, _i, _i, _p, _p, _p, _p, _i,
                                C.POINTER(_i), _p, _p, _p, _p, _p, _p]),
    "rohm_window_param_noise": (_i, [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _p, _p, _p, _p, _p, _p]),
    "rohm_window_encode_canonical": (_i, [_p, _p, _p, _i, _i, _p, _p, _p, _p, _p, _p, _p]),
    "rohm_window_to_world": (_i, [_p, _p, _p, _p, _p, _i, _i, _p, _i64, _p, _p, _p]),
    "rohm_window_encode_video": (_i, [_p, _p, _p, _p, _p, _p, C.POINTER(_i), _p, _i, _i, _i, _p, _p, _i, _p, _p, _p, _p,
                                      _i, C.POINTER(_i), _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "rohm_window_keypoints": (_i, [_p, _p, _p, _p, _p, _p, _i, _p, _p, _p, _i, _i, _p, _p, _p, _p]),
    "rohm_window_scene_joints": (_i, [_p, _p, _p, _p, _p, _p, _i, _i, _p, _p]),
    "rohm_eval_amass": (_i, [_p, _p, _p, _p, _p, _i, _p, _i, C.c_uint, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p,
                             _p]),
    "rohm_eval_video": (_i, [_p, _p, _i, _p, _p, _i, _p, _i, _p, _p, _i, _i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p]),
    "rohm_eval_reduce": (_i, [_p, _p, _i, _p, _i, _p, _p, _i, _p, _p, _p]),
}

_lock = threading.Lock()
_lib = None
_ctx = {}  # device index -> ctx pointer


def load():
    """Loads librohm_b200.so (once) and declares every prototype.  Raises RohmB200Error if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RohmB200Error(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "or `make -C rohm_b200/csrc`.  rohm_b200 has no CPU fallback.")
        try:
            lib = C.CDLL(LIB_PATH)
        except OSError as e:  # pragma: no cover
            raise RohmB200Error(f"cannot load {LIB_PATH}: {e}") from e
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def ctx(device_index):
    """The per-device rohm_ctx (created on first use)."""
    lib = load()
    if device_index in _ctx:
        return _ctx[device_index]
    with _lock:
        if device_index in _ctx:
            return _ctx[device_index]
        out = C.c_void_p()
        rc = lib.rohm_ctx_create(int(device_index), C.byref(out))
        if rc != ROHM_OK:
            raise RohmB200Error(f"rohm_ctx_create(device={device_index}) failed with status {rc}: "
                                "an sm_90 (H100) device is required; there is no CPU fallback")
        _ctx[device_index] = out
    return _ctx[device_index]


def check(rc, c):
    if rc != ROHM_OK:
        msg = load().rohm_last_error(c)
        raise RohmB200Error(f"status {rc}: {msg.decode() if msg else '?'}")
