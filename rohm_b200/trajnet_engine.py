"""Python side of the TrajNet CUDA engine: hands the module's parameters to ``rohm_trajnet_create`` by their reference
state-dict keys, tracks the step-invariant condition and runs ``rohm_trajnet_forward``."""
import ctypes as C
import os

import torch

from . import _lib
from ._lib import RohmB200Error
from .posenet import _precision_from_env


class TrajNetEngine:
    def __init__(self, module, device, max_batch, frames, precision, batch_invariant=False):
        self.lib = _lib.load()
        self.ctx = _lib.ctx(device.index)
        self.device = device
        self.max_batch, self.frames, self.precision = max_batch, frames, precision
        self.batch_invariant = batch_invariant
        sd = {k: v.detach().to(device=device, dtype=torch.float32).contiguous() for k, v in module.state_dict().items()
              if v.is_floating_point()}
        n = len(sd)
        names = (C.c_char_p * n)(*[k.encode() for k in sd])
        ptrs = (C.c_void_p * n)(*[v.data_ptr() for v in sd.values()])
        numels = (C.c_int64 * n)(*[v.numel() for v in sd.values()])
        handle = C.c_void_p()
        with torch.cuda.device(device):
            create = self.lib.rohm_trajnet_create_batch_invariant if batch_invariant else self.lib.rohm_trajnet_create
            rc = create(self.ctx, n, names, ptrs, numels, module.time_dim, module.cond_dim, module.traj_feat_dim,
                        module.mid_dim, int(module.trajcontrol), module.control_cond_dim, max_batch, frames, precision,
                        C.byref(handle))
        _lib.check(rc, self.ctx)
        self.handle = handle
        if os.environ.get("ROHM_B200_PDL", "1") == "0":
            self.lib.rohm_trajnet_set_option(handle, 1, 0)
        if os.environ.get("ROHM_B200_GRAPH", "1") == "0":
            self.lib.rohm_trajnet_set_option(handle, 0, 0)
        # strong references to the tensors whose step-invariant pyramid the engine holds (see PoseNetEngine)
        self.cond_ref, self.cond_version = None, -1
        self.control_ref, self.control_version = None, -1
        self.cond_B = -1
        self.cond_lengths = None  # the per-clip lengths the pyramid was embedded with
        self.lengths = None  # what rohm_trajnet_set_lengths last received (None: uniform clips)
        from . import ops
        self.op_key = ops.register_engine(self)
        del sd

    def __del__(self):
        h = getattr(self, "handle", None)
        try:
            from . import ops
            ops.unregister_engine(getattr(self, "op_key", 0))
        except Exception:
            pass
        if h:
            try:
                self.lib.rohm_trajnet_destroy(h)
            except Exception:
                pass
            self.handle = None

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def set_lengths(self, lengths):
        """Per-clip lengths (a tuple of ints) for the following set_cond / forward / sample_step, or None."""
        if lengths == self.lengths:
            return
        arr = None if lengths is None else (C.c_int * len(lengths))(*lengths)
        rc = self.lib.rohm_trajnet_set_lengths(self.handle, arr, 0 if lengths is None else len(lengths))
        _lib.check(rc, self.ctx)
        self.lengths = lengths

    def set_cond(self, cond, control_cond):
        rc = self.lib.rohm_trajnet_set_cond(self.handle, C.c_void_p(cond.data_ptr()),
                                            C.c_void_p(control_cond.data_ptr() if control_cond is not None else 0),
                                            cond.shape[0], self._stream())
        _lib.check(rc, self.ctx)

    def forward(self, x_t, time):
        """The denoiser call, through the custom op torch.ops.rohm.trajnet_forward."""
        return torch.ops.rohm.trajnet_forward(self.op_key, x_t, time)

    def _forward_impl(self, x_t, time):
        out = torch.empty_like(x_t)
        rc = self.lib.rohm_trajnet_forward(self.handle, C.c_void_p(x_t.data_ptr()), C.c_void_p(time.data_ptr()),
                                           C.c_void_p(out.data_ptr()), x_t.shape[0], self._stream())
        _lib.check(rc, self.ctx)
        return out

    def sample_step(self, x_t, time, coef_row, streams=None):
        """One whole ancestral step as one graph launch (rohm_trajnet_sample_step): -> (pred_xstart, x_{t-1}); the noise is
        what torch.randn_like(x_t) would have drawn (torch's CUDA generator is advanced accordingly).  streams
        (noise_streams.NoiseStreams): clip b's noise comes from its own generator instead (rohm_trajnet_sample_step_clips),
        over the engine's current lengths, and x_{t-1} is zero past each clip."""
        from .ops import cuda_generator_state
        x0, nxt = torch.empty_like(x_t), torch.empty_like(x_t)
        if streams is not None:
            draw = streams.next_draw((x_t.shape[2], x_t.shape[1], True, self.lengths))
            rc = self.lib.rohm_trajnet_sample_step_clips(self.handle, C.c_void_p(x_t.data_ptr()), C.c_void_p(time.data_ptr()),
                                                         C.c_void_p(x0.data_ptr()), C.c_void_p(nxt.data_ptr()),
                                                         C.c_void_p(coef_row.data_ptr()),
                                                         C.c_void_p(streams.table.data_ptr()), draw, streams.incs,
                                                         x_t.shape[0], self._stream())
            _lib.check(rc, self.ctx)
            return x0, nxt
        gen, seed, offset = cuda_generator_state(x_t.device)
        inc = C.c_uint64(0)
        rc = self.lib.rohm_trajnet_sample_step(self.handle, C.c_void_p(x_t.data_ptr()), C.c_void_p(time.data_ptr()),
                                               C.c_void_p(x0.data_ptr()), C.c_void_p(nxt.data_ptr()),
                                               C.c_void_p(coef_row.data_ptr()), seed, offset, C.byref(inc), x_t.shape[0],
                                               self._stream())
        _lib.check(rc, self.ctx)
        gen.set_offset(offset + int(inc.value))
        return x0, nxt

    @property
    def launches_per_forward(self):
        return int(self.lib.rohm_trajnet_launches_per_forward(self.handle))


def _fingerprint(module):
    return tuple((p.data_ptr(), p._version) for p in module.parameters())


def _f32c(t):
    return t if (t.is_contiguous() and t.dtype == torch.float32) else t.contiguous().float()


def get_engine(module, B, T, device):
    if module.training:
        raise RohmB200Error("TrajNet: the CUDA engine implements the inference path (model.eval()); training is out of "
                            "scope")
    prec = module.precision if module.precision is not None else _precision_from_env()
    inv = batch_invariant(module)
    e = module._engine
    if e is None or e.device != device or B > e.max_batch or T != e.frames or e.precision != prec or \
            e.batch_invariant != inv:
        mb = max(B, e.max_batch if (e is not None and e.device == device and e.frames == T) else 0)
        module._engine = None
        e = TrajNetEngine(module, device, mb, T, prec, inv)
        module._engine = e
        module._engine_fingerprint = _fingerprint(module)
    return e


def batch_invariant(module):
    """module.batch_invariant, checked: a bool (absent on modules built before the attribute existed: False)."""
    v = getattr(module, 'batch_invariant', False)
    if not isinstance(v, bool):
        raise RohmB200Error(f"TrajNet: batch_invariant must be True or False, got {v!r}")
    return v


def prepare(module, batch, time):
    """Argument checks, engine lookup and the step-invariant condition pyramid of one denoiser call: -> (engine, x_t as a
    contiguous fp32 tensor, time as contiguous int64)."""
    x_t, cond = batch['x_t'], batch['cond']
    if x_t.device.type != "cuda":
        raise RohmB200Error("TrajNet: batch tensors must live on a CUDA device (no CPU path)")
    if x_t.dim() != 3 or x_t.shape[-1] != module.traj_feat_dim or cond.shape[:2] != x_t.shape[:2] or \
            cond.shape[-1] != module.cond_dim:
        raise RohmB200Error(f"TrajNet: expected x_t [B, T, {module.traj_feat_dim}] and cond [B, T, {module.cond_dim}], "
                            f"got {tuple(x_t.shape)} / {tuple(cond.shape)}")
    B, T, _ = x_t.shape
    if T % 16 != 0:
        raise RohmB200Error(f"TrajNet: the number of frames ({T}) must be a multiple of 16 (four stride-2 stages)")
    control = batch.get('control_cond') if module.trajcontrol else None
    if module.trajcontrol and (control is None or tuple(control.shape) != (B, T, module.control_cond_dim)):
        raise RohmB200Error(f"TrajNet(trajcontrol=True): batch['control_cond'] must be [B, T, {module.control_cond_dim}]")
    lengths = clip_lengths(batch, x_t.shape) if batch.get('lengths') is not None else None
    e = get_engine(module, B, T, x_t.device)
    # object identity + version (never data_ptr: freed addresses are recycled by the caching allocator)
    same = (e.cond_ref is cond and e.cond_version == cond._version and e.cond_B == B and e.control_ref is control and
            (control is None or e.control_version == control._version) and e.cond_lengths == lengths)
    if not same:
        if _fingerprint(module) != module._engine_fingerprint:  # parameters changed since the weights were packed
            module._engine = None
            e = get_engine(module, B, T, x_t.device)
        e.set_lengths(lengths)
        e.set_cond(_f32c(cond), _f32c(control) if control is not None else None)
        e.cond_ref, e.cond_version, e.cond_B, e.cond_lengths = cond, cond._version, B, lengths
        e.control_ref, e.control_version = control, (control._version if control is not None else -1)
    ts = time.to(device=x_t.device, dtype=torch.int64).contiguous()
    return e, _f32c(x_t), ts


def clip_lengths(batch, shape):
    """batch['lengths'] checked against the padded [B, T, *] batch `shape`, as a tuple of ints; None when the key is absent.
    Raises RohmB200Error before anything runs on the device."""
    lengths = batch.get('lengths') if isinstance(batch, dict) else None
    if lengths is None:
        return None
    B, T = int(shape[0]), int(shape[1])
    if (not isinstance(lengths, torch.Tensor) or lengths.is_floating_point() or lengths.is_complex() or
            lengths.dtype == torch.bool or tuple(lengths.shape) != (B,)):
        raise RohmB200Error(f"TrajNet: batch['lengths'] must be an integer tensor of shape [{B}], got "
                            f"{getattr(lengths, 'dtype', type(lengths))} {tuple(getattr(lengths, 'shape', ()))}")
    values = tuple(int(v) for v in lengths.tolist())
    bad = [(b, v) for b, v in enumerate(values) if not (16 <= v <= T and v % 16 == 0)]
    if bad:
        raise RohmB200Error(f"TrajNet: batch['lengths'] must be multiples of 16 in [16, T={T}] (four stride-2 stages); "
                            f"lengths[{bad[0][0]}] = {bad[0][1]}")
    return values
