"""PyTorch-facing operators: thin checked wrappers that hand raw device pointers and the current CUDA stream to the
C-ABI library.  PyTorch is plumbing here (device memory, streams); all arithmetic happens in librohm_b200.so.

The elementwise sampler ops are also registered as ``torch.ops.rohm.*`` custom ops.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import RohmB200Error


def _require_cuda(name, t, dtype=torch.float32):
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise RohmB200Error(f"{name}: expected a CUDA tensor (rohm_b200 has no CPU path), got "
                            f"{getattr(t, 'device', type(t))}")
    if t.dtype != dtype:
        raise RohmB200Error(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise RohmB200Error(f"{name}: tensor must be contiguous")


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _update_args(name, x0, x_t, coef, grads, noise=None):
    """The checks the update wrappers share, all before any launch: -> (B, elements per clip, coef stride, grad 0,
    grad 1).  coef is one shared row [8] (stride 0) or one row per clip [B, 8]; at most two guidance gradients."""
    tensors = (("x0", x0), ("x_t", x_t)) + ((("noise", noise),) if noise is not None else ()) + (("coef", coef),)
    for n, t in tensors:
        _require_cuda(n, t)
    if x0.shape != x_t.shape or (noise is not None and noise.shape != x0.shape):
        raise RohmB200Error(f"{name}: {'x0, x_t and noise' if noise is not None else 'x0 and x_t'} must have the same "
                            "shape")
    for g in grads:
        _require_cuda("grad", g)
        if g.shape != x0.shape:
            raise RohmB200Error(f"{name}: grad shape mismatch")
    B = x0.shape[0]
    if coef.dim() == 1:
        if coef.numel() < _lib.DDPM_COEFS:
            raise RohmB200Error(f"{name}: coef row must hold 8 floats")
        stride = 0
    elif coef.shape != (B, _lib.DDPM_COEFS):
        raise RohmB200Error(f"{name}: per-clip coef must be [{B}, 8]")
    else:
        stride = _lib.DDPM_COEFS
    return B, x0.numel() // max(B, 1), stride, (grads[0] if grads else None), (grads[1] if len(grads) > 1 else None)


def ddpm_step(x0, x_t, noise, coef, grads=(), out=None):
    """out = c1*x0 + c2*x_t (+ gs_k*grad_k) + sigma*noise; coef: fp32 CUDA [8] (shared) or [B, 8] (per clip)."""
    B, clip_elems, stride, g0, g1 = _update_args("ddpm_step", x0, x_t, coef, grads, noise)
    if out is None:
        out = torch.empty_like(x0)
    lib, c = _lib.load(), _lib.ctx(x0.device.index)
    rc = lib.rohm_ddpm_step(c, _ptr(x0), _ptr(x_t), _ptr(noise), _ptr(g0), _ptr(g1), len(grads), _ptr(out), B,
                            clip_elems, _ptr(coef), stride, _stream(x0.device))
    _lib.check(rc, c)
    return out


def cuda_generator_state(device):
    """(generator, seed, offset) of torch's default CUDA generator of `device`: what torch.randn_like would consume next."""
    gen = torch.cuda.default_generators[device.index if device.index is not None else torch.cuda.current_device()]
    return gen, int(gen.initial_seed()), int(gen.get_offset())


def ddpm_step_philox(x0, x_t, coef, grads=(), out=None):
    """ddpm_step with noise = torch.randn_like(x_t) drawn inside the kernel from torch's CUDA generator (same values, same
    generator advance as the explicit call), saving the noise tensor's launch and its HBM round trip."""
    B, clip_elems, stride, g0, g1 = _update_args("ddpm_step_philox", x0, x_t, coef, grads)
    if out is None:
        out = torch.empty_like(x0)
    lib, c = _lib.load(), _lib.ctx(x0.device.index)
    gen, seed, offset = cuda_generator_state(x0.device)
    inc = C.c_uint64(0)
    rc = lib.rohm_ddpm_step_philox(c, _ptr(x0), _ptr(x_t), _ptr(g0), _ptr(g1), len(grads), _ptr(out), B, clip_elems,
                                   _ptr(coef), stride, seed, offset, C.byref(inc), _stream(x0.device))
    _lib.check(rc, c)
    gen.set_offset(offset + int(inc.value))
    return out


def _clip_layout(shape, channels_last):
    """(B, C, T) of a padded PoseNet [B, C, 1, T] (channels_last=False) or TrajNet [B, T, C] (channels_last=True) batch."""
    if channels_last:
        if len(shape) != 3:
            raise RohmB200Error(f"per-clip noise: a channels-last batch is [B, T, C], got {tuple(shape)}")
        return int(shape[0]), int(shape[2]), int(shape[1])
    if len(shape) != 4 or shape[2] != 1:
        raise RohmB200Error(f"per-clip noise: a channel-major batch is [B, C, 1, T], got {tuple(shape)}")
    return int(shape[0]), int(shape[1]), int(shape[3])


def randn_clips(streams, shape, channels_last, lengths=None, device=None):
    """A padded batch of `shape` whose clip b holds torch.randn(S_b, generator=streams.generators[b]) in its real frames
    (lengths[b], or all T) and zero past them (rohm_randn_clips).  streams: noise_streams.NoiseStreams."""
    B, Cc, T = _clip_layout(shape, channels_last)
    if B != len(streams):
        raise RohmB200Error(f"randn_clips: {len(streams)} streams for a batch of {B} clips")
    dev = streams.table.device if device is None else torch.device(device)
    out = torch.empty(tuple(shape), device=dev, dtype=torch.float32)
    draw = streams.next_draw((Cc, T, bool(channels_last), lengths))
    lib, c = _lib.load(), _lib.ctx(out.device.index)
    rc = lib.rohm_randn_clips(c, _ptr(out), B, Cc, T, int(bool(channels_last)), streams.lengths_c(lengths),
                              _ptr(streams.table), draw, streams.incs, _stream(out.device))
    _lib.check(rc, c)
    return out


def ddpm_step_philox_clips(x0, x_t, coef, streams, channels_last, lengths=None, grads=(), out=None):
    """ddpm_step with noise = randn_clips(streams, x_t.shape, channels_last, lengths) drawn inside the kernel (same bits),
    and zero in every clip's padded frames."""
    _, _, stride, g0, g1 = _update_args("ddpm_step_philox_clips", x0, x_t, coef, grads)
    B, Cc, T = _clip_layout(x0.shape, channels_last)
    if B != len(streams):
        raise RohmB200Error(f"ddpm_step_philox_clips: {len(streams)} streams for a batch of {B} clips")
    if out is None:
        out = torch.empty_like(x0)
    draw = streams.next_draw((Cc, T, bool(channels_last), lengths))
    lib, c = _lib.load(), _lib.ctx(x0.device.index)
    rc = lib.rohm_ddpm_step_philox_clips(c, _ptr(x0), _ptr(x_t), _ptr(g0), _ptr(g1), len(grads), _ptr(out), B, Cc, T,
                                         int(bool(channels_last)), streams.lengths_c(lengths), _ptr(coef), stride,
                                         _ptr(streams.table), draw, streams.incs, _stream(x0.device))
    _lib.check(rc, c)
    return out


def q_sample(x_start, noise, sqrt_ac, sqrt_one_minus_ac):
    _require_cuda("x_start", x_start)
    _require_cuda("noise", noise)
    out = torch.empty_like(x_start)
    lib, c = _lib.load(), _lib.ctx(x_start.device.index)
    rc = lib.rohm_q_sample(c, _ptr(x_start), _ptr(noise), _ptr(out), x_start.numel(), float(sqrt_ac),
                           float(sqrt_one_minus_ac), _stream(x_start.device))
    _lib.check(rc, c)
    return out


def ddim_step(x0, x_t, noise, coefs):
    for n, t in (("x0", x0), ("x_t", x_t), ("noise", noise)):
        _require_cuda(n, t)
    out = torch.empty_like(x0)
    lib, c = _lib.load(), _lib.ctx(x0.device.index)
    sr, srm1, sap, dirc, sigma = coefs
    rc = lib.rohm_ddim_step(c, _ptr(x0), _ptr(x_t), _ptr(noise), _ptr(out), x0.numel(), sr, srm1, sap, dirc, sigma,
                            _stream(x0.device))
    _lib.check(rc, c)
    return out


# ---------------------------------------------------------------------------------------------------------------
# torch.library registration (torch.ops.rohm.*)
# ---------------------------------------------------------------------------------------------------------------
# Engine objects (PoseNetEngine / TrajNetEngine / BodyKernels: one C handle + workspace each) are addressed by an integer
# key, so the denoiser and body-model entry points are ordinary tensor-in / tensor-out custom ops as well.
_engines = {}


def register_engine(engine):
    import weakref
    key = id(engine)
    _engines[key] = weakref.ref(engine)  # weak: the registry must not keep a replaced engine (and its device memory) alive
    return key


def unregister_engine(key):
    _engines.pop(key, None)


def _engine(key):
    ref = _engines.get(int(key))
    e = ref() if ref is not None else None
    if e is None:
        raise RohmB200Error(f"torch.ops.rohm: unknown engine key {key} (engine destroyed?)")
    return e


try:
    @torch.library.custom_op("rohm::posenet_forward", mutates_args=(), device_types="cuda")
    def _posenet_forward_op(engine: int, x_t: torch.Tensor, timesteps: torch.Tensor) -> torch.Tensor:
        return _engine(engine)._forward_impl(x_t, timesteps)

    @_posenet_forward_op.register_fake
    def _(engine, x_t, timesteps):
        return torch.empty_like(x_t)

    @torch.library.custom_op("rohm::trajnet_forward", mutates_args=(), device_types="cuda")
    def _trajnet_forward_op(engine: int, x_t: torch.Tensor, time: torch.Tensor) -> torch.Tensor:
        return _engine(engine)._forward_impl(x_t, time)

    @_trajnet_forward_op.register_fake
    def _(engine, x_t, time):
        return torch.empty_like(x_t)

    @torch.library.custom_op("rohm::skating_guidance", mutates_args=(), device_types="cuda")
    def _skating_guidance_op(engine: int, x0: torch.Tensor, mean: torch.Tensor, std: torch.Tensor) -> torch.Tensor:
        return _engine(engine).skating_guidance(x0, mean, std)

    @_skating_guidance_op.register_fake
    def _(engine, x0, mean, std):
        return torch.empty_like(x0)

    @torch.library.custom_op("rohm::ddpm_step_philox", mutates_args=(), device_types="cuda")
    def _ddpm_step_philox_op(x0: torch.Tensor, x_t: torch.Tensor, coef: torch.Tensor) -> torch.Tensor:
        return ddpm_step_philox(x0, x_t, coef)

    @_ddpm_step_philox_op.register_fake
    def _(x0, x_t, coef):
        return torch.empty_like(x0)
except Exception:  # pragma: no cover
    pass

try:
    @torch.library.custom_op("rohm::ddpm_step", mutates_args=(), device_types="cuda")
    def _ddpm_step_op(x0: torch.Tensor, x_t: torch.Tensor, noise: torch.Tensor, coef: torch.Tensor) -> torch.Tensor:
        return ddpm_step(x0, x_t, noise, coef)

    @_ddpm_step_op.register_fake
    def _(x0, x_t, noise, coef):
        return torch.empty_like(x0)

    @torch.library.custom_op("rohm::q_sample", mutates_args=(), device_types="cuda")
    def _q_sample_op(x_start: torch.Tensor, noise: torch.Tensor, a: float, b: float) -> torch.Tensor:
        return q_sample(x_start, noise, a, b)

    @_q_sample_op.register_fake
    def _(x_start, noise, a, b):
        return torch.empty_like(x_start)
except Exception:  # pragma: no cover - registration is a convenience, the python entry points above are the API
    pass
