"""PoseNet: drop-in for reference model/posenet.py:11-96 (constructor, attributes, state-dict keys, call signature),
with the forward pass executed by the CUDA engine behind ``rohm_posenet_*`` (include/rohm_b200.h).

The module owns its parameters in torch containers named exactly like the reference so ``load_state_dict(strict=True)``
works on released checkpoints; on the first forward (and whenever parameters change) they are repacked into the
engine's TF32 hi/lo layout.  There is no eager / CPU forward: calling the model without an H100 raises.
"""
import ctypes as C
import os

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from ._lib import RohmB200Error
from .heads import InputProcess, OutputProcess, PositionalEncoding, TimestepEmbedder


DEFAULT_PRECISION = "f16x2"


def _precision_from_env(supports_f16=True):
    """ROHM_B200_PRECISION: 'f16x2' (default: fp16 hi/lo pairs, fp32-grade), 'tf32x3' (TF32 hi/lo pairs, fp32-grade),
    'tf32' (single pass, fast, ~1e-3).  Engines without an fp16 path (the LBS blend GEMM) run 'f16x2' as 'tf32x3'."""
    v = os.environ.get("ROHM_B200_PRECISION", DEFAULT_PRECISION).lower()
    if v in ("f16x2", "fp16x2", "parity"):
        return _lib.PRECISION_F16X2 if supports_f16 else _lib.PRECISION_TF32X3
    if v in ("tf32x3", "3xtf32", "fp32"):
        return _lib.PRECISION_TF32X3
    if v in ("tf32", "fast"):
        return _lib.PRECISION_TF32
    raise RohmB200Error(f"ROHM_B200_PRECISION={v!r}: expected 'f16x2' (default), 'tf32x3' or 'tf32' (fast)")


class PoseNetEngine:
    """Owns one rohm_posenet handle (device weights + workspace) sized for (max_batch, max_frames)."""

    def __init__(self, module, device, max_batch, max_frames, precision):
        self.lib = _lib.load()
        self.ctx = _lib.ctx(device.index)
        self.device = device
        self.max_batch, self.max_frames, self.precision = max_batch, max_frames, precision
        sd = {k: v.detach().to(device=device, dtype=torch.float32).contiguous() for k, v in module.state_dict().items()
              if not k.startswith("smplx_model.")}
        self._keep = sd  # keeps the source tensors alive during create (the library copies them)
        L = module.num_layers
        layers = (_lib.PoseNetLayerW * L)()
        for l in range(L):
            p = f"seqTransEncoder.layers.{l}."
            for field, key in (("in_proj_w", "self_attn.in_proj_weight"), ("in_proj_b", "self_attn.in_proj_bias"),
                               ("out_proj_w", "self_attn.out_proj.weight"), ("out_proj_b", "self_attn.out_proj.bias"),
                               ("lin1_w", "linear1.weight"), ("lin1_b", "linear1.bias"),
                               ("lin2_w", "linear2.weight"), ("lin2_b", "linear2.bias"),
                               ("norm1_w", "norm1.weight"), ("norm1_b", "norm1.bias"),
                               ("norm2_w", "norm2.weight"), ("norm2_b", "norm2.bias")):
                setattr(layers[l], field, sd[p + key].data_ptr())
        pe = sd["sequence_pos_encoder.pe"].reshape(-1, module.latent_dim).contiguous()
        self._keep["__pe2d"] = pe
        w = _lib.PoseNetW()
        w.d_model, w.ff_size, w.num_layers, w.num_heads = module.latent_dim, module.ff_size, L, module.num_heads
        w.in_feats, w.out_feats, w.traj_feats = module.input_feats, module.output_process.output_feats, module.traj_feat_dim
        w.pe_len = pe.shape[0]
        for field, key in (("in_w", "input_process.poseEmbedding.weight"), ("in_b", "input_process.poseEmbedding.bias"),
                           ("cond_w", "input_process_cond.poseEmbedding.weight"),
                           ("cond_b", "input_process_cond.poseEmbedding.bias"),
                           ("t0_w", "embed_timestep.time_embed.0.weight"), ("t0_b", "embed_timestep.time_embed.0.bias"),
                           ("t2_w", "embed_timestep.time_embed.2.weight"), ("t2_b", "embed_timestep.time_embed.2.bias"),
                           ("out_w", "output_process.poseFinal.weight"), ("out_b", "output_process.poseFinal.bias")):
            setattr(w, field, sd[key].data_ptr())
        w.pe = pe.data_ptr()
        w.layers = layers
        if w.in_feats != w.traj_feats + w.out_feats:
            raise RohmB200Error(f"PoseNet: body_feat_dim ({w.in_feats}) must equal traj_feat_dim ({w.traj_feats}) + "
                                f"pose_feat_dim ({w.out_feats})")
        handle = C.c_void_p()
        with torch.cuda.device(device):
            rc = self.lib.rohm_posenet_create(self.ctx, C.byref(w), max_batch, max_frames, precision, C.byref(handle))
        _lib.check(rc, self.ctx)
        self.handle = handle
        self._keep = None  # the library owns its copies now
        if os.environ.get("ROHM_B200_PDL", "1") == "0":
            self.lib.rohm_posenet_set_option(handle, 1, 0)
        if os.environ.get("ROHM_B200_GRAPH", "1") == "0":
            self.lib.rohm_posenet_set_option(handle, 0, 0)
        # the condition whose step-invariant embedding the engine currently holds: a STRONG reference (so the caching
        # allocator cannot hand its address to a different tensor while it is cached), its version counter and the
        # per-clip lengths it was embedded with
        self.cond_ref = None
        self.cond_version = -1
        self.cond_lengths = None
        self.lengths = None  # what rohm_posenet_set_lengths last received (None: uniform clips)
        from . import ops
        self.op_key = ops.register_engine(self)

    def __del__(self):
        h = getattr(self, "handle", None)
        try:
            from . import ops
            ops.unregister_engine(getattr(self, "op_key", 0))
        except Exception:
            pass
        if h:
            try:
                self.lib.rohm_posenet_destroy(h)
            except Exception:
                pass
            self.handle = None

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def set_lengths(self, lengths):
        """Per-clip lengths (a tuple of ints) for the following set_cond / forward / sample_step / profile, or None."""
        if lengths == self.lengths:
            return
        arr = None if lengths is None else (C.c_int * len(lengths))(*lengths)
        rc = self.lib.rohm_posenet_set_lengths(self.handle, arr, 0 if lengths is None else len(lengths))
        _lib.check(rc, self.ctx)
        self.lengths = lengths

    def set_cond(self, cond):
        B, _, _, T = cond.shape
        rc = self.lib.rohm_posenet_set_cond(self.handle, C.c_void_p(cond.data_ptr()), B, T, self._stream())
        _lib.check(rc, self.ctx)

    def forward(self, x_t, timesteps, out=None):
        """The denoiser call, through the custom op torch.ops.rohm.posenet_forward (an explicit `out` skips the op layer)."""
        if out is None:
            return torch.ops.rohm.posenet_forward(self.op_key, x_t, timesteps)
        return self._forward_impl(x_t, timesteps, out)

    def _forward_impl(self, x_t, timesteps, out=None):
        B, _, _, T = x_t.shape
        if out is None:
            out = torch.empty_like(x_t)
        rc = self.lib.rohm_posenet_forward(self.handle, C.c_void_p(x_t.data_ptr()), C.c_void_p(timesteps.data_ptr()),
                                           C.c_void_p(out.data_ptr()), B, T, self._stream())
        _lib.check(rc, self.ctx)
        return out

    def sample_step(self, x_t, timesteps, coef_row, streams=None):
        """One whole ancestral step as one graph launch (rohm_posenet_sample_step): -> (pred_xstart, x_{t-1}); the noise is
        what torch.randn_like(x_t) would have drawn (torch's CUDA generator is advanced accordingly).  streams
        (noise_streams.NoiseStreams): clip b's noise comes from its own generator instead (rohm_posenet_sample_step_clips),
        over the engine's current lengths, and x_{t-1} is zero past each clip."""
        from .ops import cuda_generator_state
        B, C_, _, T = x_t.shape
        x0, nxt = torch.empty_like(x_t), torch.empty_like(x_t)
        if streams is not None:
            draw = streams.next_draw((C_, T, False, self.lengths))
            rc = self.lib.rohm_posenet_sample_step_clips(self.handle, C.c_void_p(x_t.data_ptr()),
                                                         C.c_void_p(timesteps.data_ptr()), C.c_void_p(x0.data_ptr()),
                                                         C.c_void_p(nxt.data_ptr()), C.c_void_p(coef_row.data_ptr()),
                                                         C.c_void_p(streams.table.data_ptr()), draw, streams.incs, B, T,
                                                         self._stream())
            _lib.check(rc, self.ctx)
            return x0, nxt
        gen, seed, offset = cuda_generator_state(x_t.device)
        inc = C.c_uint64(0)
        rc = self.lib.rohm_posenet_sample_step(self.handle, C.c_void_p(x_t.data_ptr()), C.c_void_p(timesteps.data_ptr()),
                                               C.c_void_p(x0.data_ptr()), C.c_void_p(nxt.data_ptr()),
                                               C.c_void_p(coef_row.data_ptr()), seed, offset, C.byref(inc), B, T, self._stream())
        _lib.check(rc, self.ctx)
        gen.set_offset(offset + int(inc.value))
        return x0, nxt

    def profile(self, x_t, timesteps):
        """One forward with per-kernel CUDA-event timing -> ({category: ms}, {category: launches})."""
        B, _, _, T = x_t.shape
        out = torch.empty_like(x_t)
        ms = (C.c_float * 4)()
        n = (C.c_int * 4)()
        rc = self.lib.rohm_posenet_profile(self.handle, C.c_void_p(x_t.data_ptr()), C.c_void_p(timesteps.data_ptr()),
                                           C.c_void_p(out.data_ptr()), B, T, self._stream(), ms, n)
        _lib.check(rc, self.ctx)
        names = ("gemm", "attention", "layernorm", "other")
        return {k: float(ms[i]) for i, k in enumerate(names)}, {k: int(n[i]) for i, k in enumerate(names)}

    @property
    def launches_per_forward(self):
        return int(self.lib.rohm_posenet_launches_per_forward(self.handle))


def _create_body_model(body_model_path, device):
    """The SMPL-X body model submodule (reference posenet.py:57-58).  Uses the real ``smplx`` package when it is
    installed (so checkpoint keys under ``smplx_model.*`` match); otherwise the package's own BodyModel."""
    try:
        import smplx  # noqa: F401  third-party, optional
        m = smplx.create(model_path=body_model_path, model_type="smplx", gender='neutral', flat_hand_mean=True,
                         use_pca=False)
        return m.to(device) if device is not None else m
    except ImportError:
        from .body_model import BodyModel
        return BodyModel.create(body_model_path, device=device)


class PoseNet(nn.Module):
    def __init__(self, dataset, body_feat_dim, nfeats=1,
                 latent_dim=256, ff_size=1024, num_layers=8, num_heads=4, dropout=0.1, activation="gelu",
                 body_model_path='',
                 device=None,
                 traj_feat_dim=4,
                 weight_loss_rec_repr_full_body=0.0,
                 weight_loss_repr_foot_contact_mse=0.0,
                 weight_loss_joint_pos_global=0.0,
                 weight_loss_joint_vel_global=0.0, weight_loss_joint_smooth=0.0,
                 weight_loss_foot_skating=0.0,
                 start_skating_loss_epoch=0,
                 ):
        super().__init__()
        if activation != "gelu":
            raise RohmB200Error("PoseNet: only activation='gelu' (the configuration RoHM ships) is implemented")
        self.dataset = dataset
        self.body_feat_dim = body_feat_dim
        self.nfeats = nfeats
        self.traj_feat_dim = traj_feat_dim
        self.foot_joint_index_list = [7, 10, 8, 11]  # left ankle, left toe, right ankle, right toe
        self.foot_skating_vel_thres = 0.1
        self.fps = 30
        self.latent_dim = latent_dim
        self.ff_size = ff_size
        self.num_layers = num_layers
        self.num_heads = num_heads
        self.dropout = dropout
        self.activation = activation
        self.input_feats = self.body_feat_dim * self.nfeats
        self.normalize_output = False
        self.device = device
        self.weight_loss_rec_repr_full_body = weight_loss_rec_repr_full_body
        self.weight_loss_repr_foot_contact_mse = weight_loss_repr_foot_contact_mse
        self.weight_loss_joint_pos_global = weight_loss_joint_pos_global
        self.weight_loss_joint_vel_global = weight_loss_joint_vel_global
        self.weight_loss_joint_smooth = weight_loss_joint_smooth
        self.weight_loss_foot_skating = weight_loss_foot_skating
        self.start_skating_loss_epoch = start_skating_loss_epoch

        self.smplx_model = _create_body_model(body_model_path, device)
        self.input_process = InputProcess(self.input_feats, self.latent_dim)
        self.input_process_cond = InputProcess(self.input_feats, self.latent_dim)
        self.sequence_pos_encoder = PositionalEncoding(self.latent_dim, self.dropout)
        enc_layer = nn.TransformerEncoderLayer(d_model=self.latent_dim, nhead=self.num_heads,
                                               dim_feedforward=self.ff_size, dropout=self.dropout,
                                               activation=self.activation)
        self.seqTransEncoder = nn.TransformerEncoder(enc_layer, num_layers=self.num_layers,
                                                     enable_nested_tensor=False)
        self.embed_timestep = TimestepEmbedder(self.latent_dim, self.sequence_pos_encoder)
        self.output_process = OutputProcess(self.dataset.pose_feat_dim, self.latent_dim, self.nfeats)

        self.precision = None  # None -> ROHM_B200_PRECISION env (default f16x2)
        # test-time guidance loss normalisers: 'batch' (the reference on the whole batch) or 'clip' (each clip as the
        # reference on that clip alone); see guidance_per_clip
        self.guidance_normaliser = 'batch'
        self._engine = None
        self._engine_fingerprint = None

    # ---------------------------------------------------------------- engine management
    def _fingerprint(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def invalidate_engine(self):
        """Forces the weights to be repacked on the next forward (call after mutating parameters in place)."""
        self._engine = None

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict=True, **k):
        """nn.Module.load_state_dict, plus: when the body model is the package's own BodyModel (no ``smplx`` package
        installed), the ``smplx_model.*`` entries of a reference checkpoint are adopted by buffer name
        (BodyModel.load_smplx_state) instead of being matched key by key -- real smplx registers more buffers than
        RoHM's calls need, so a strict key match could never succeed."""
        self._engine = None
        from .body_model import BodyModel
        if isinstance(self.smplx_model, BodyModel):
            prefix = "smplx_model."
            body = {key[len(prefix):]: v for key, v in state_dict.items() if key.startswith(prefix)}
            rest = {key: v for key, v in state_dict.items() if not key.startswith(prefix)}
            own = {prefix + n: b for n, b in self.smplx_model.state_dict().items()}
            foreign = [n for n in body if (prefix + n) not in own or own[prefix + n].shape != body[n].shape]
            if foreign:
                self.smplx_model.load_smplx_state(body)
                rest.update({prefix + n: b for n, b in self.smplx_model.state_dict().items()})
            else:
                rest.update({prefix + n: v for n, v in body.items()})
                for key, v in own.items():
                    rest.setdefault(key, v)
            state_dict = rest
        return super().load_state_dict(state_dict, strict=strict, **k)

    def engine(self, B, T, device):
        if self.training:
            raise RohmB200Error("PoseNet: the CUDA engine implements the inference path (model.eval()); training is "
                                "out of scope")
        prec = self.precision if self.precision is not None else _precision_from_env()
        e = self._engine
        if (e is None or e.device != device or B > e.max_batch or T > e.max_frames or e.precision != prec):
            mb = max(B, e.max_batch if e is not None and e.device == device else 0)
            mf = max(T, e.max_frames if e is not None and e.device == device else 0)
            self._engine = None
            e = PoseNetEngine(self, device, mb, mf, prec)
            self._engine = e
            self._engine_fingerprint = self._fingerprint()
        return e

    def prepare_cond(self, cond, lengths=None):
        """Runs the step-invariant part of the forward for this condition tensor if it is new or was modified, or if the
        per-clip lengths (a tuple from clip_lengths, or None) differ from those it was embedded with."""
        if cond.device.type != "cuda":
            raise RohmB200Error("PoseNet: batch tensors must live on a CUDA device (no CPU path)")
        B, Cc, _, T = cond.shape
        e = self.engine(B, T, cond.device)
        # Same tensor OBJECT, unmodified since it was embedded -> reuse.  Identity (not data_ptr): a freed condition's
        # address and version count can be handed to the next batch's tensor by the caching allocator.
        if e.cond_ref is not cond or e.cond_version != cond._version or e.cond_lengths != lengths:
            fp = self._fingerprint()  # parameters are re-checked once per new condition, not per step
            if fp != self._engine_fingerprint:
                self._engine = None
                e = self.engine(B, T, cond.device)
            c = cond if (cond.is_contiguous() and cond.dtype == torch.float32) else cond.contiguous().float()
            e.set_lengths(lengths)
            e.set_cond(c)
            e.cond_ref, e.cond_version, e.cond_lengths = cond, cond._version, lengths
        return e

    def clip_lengths(self, batch, shape=None, grad_type=None):
        """batch['lengths'] checked against the padded [B, C, 1, T] batch (`shape`, else batch['cond'] / batch['x_t']) and
        this configuration, as a tuple of ints; None when the key is absent.  Raises RohmB200Error before anything runs on
        the device.  grad_type: the sampling loop's guidance, refused where lengths are not supported."""
        lengths = batch.get('lengths') if isinstance(batch, dict) else None
        if lengths is None:
            return None
        if shape is None:
            shape = (batch['cond'] if 'cond' in batch else batch['x_t']).shape
        B, T = int(shape[0]), int(shape[-1])
        cache = getattr(self, "_lengths_cache", None)
        if cache is not None and cache[0] is lengths and cache[1] == lengths._version and cache[2] == (B, T):
            values = cache[3]
        else:
            if (not isinstance(lengths, torch.Tensor) or lengths.is_floating_point() or lengths.is_complex() or
                    lengths.dtype == torch.bool or tuple(lengths.shape) != (B,)):
                raise RohmB200Error(f"PoseNet: batch['lengths'] must be an integer tensor of shape [{B}], got "
                                    f"{getattr(lengths, 'dtype', type(lengths))} {tuple(getattr(lengths, 'shape', ()))}")
            values = tuple(int(v) for v in lengths.tolist())
            bad = [(b, v) for b, v in enumerate(values) if not 1 <= v <= T]
            if bad:
                raise RohmB200Error(f"PoseNet: batch['lengths'] must lie in [1, T={T}]; lengths[{bad[0][0]}] = {bad[0][1]}")
            self._lengths_cache = (lengths, lengths._version, (B, T), values)
        out_of_scope = None
        per_clip = self.guidance_per_clip() if grad_type is not None else False
        prec = self.precision if self.precision is not None else _precision_from_env()
        if prec != _lib.PRECISION_F16X2:
            out_of_scope = "the tf32x3 / tf32 precisions"
        elif self.latent_dim // self.num_heads != 128:
            out_of_scope = f"head dim {self.latent_dim // self.num_heads}"
        elif grad_type == 'prox' and not per_clip:
            out_of_scope = "grad_type='prox' (2-D projection guidance)"
        elif grad_type is not None and getattr(self, "guidance_sum_reducer", None) is not None:
            out_of_scope = "parallel.global_guidance (the exact-global sharded skating normaliser)"
        if out_of_scope is not None:
            raise RohmB200Error(f"PoseNet: batch['lengths'] with {out_of_scope} is out of scope; per-clip lengths run "
                                "with precision f16x2, head dim 128 and the skating guidance only (both guidance terms "
                                "with guidance_normaliser='clip')")
        return values

    def guidance_per_clip(self):
        """Whether the guidance terms are normalised per clip (guidance_normaliser='clip'): clip b's skating and 2-D
        projection terms are then the reference's on clip b alone, a [1, 294, 1, n_b] batch (n_b = lengths[b] or T), so a
        guided recording samples the same in any batch.  'batch' (the default) normalises over the whole batch as the
        reference does.  Raises RohmB200Error, before anything runs on the device, for any other value and for 'clip'
        together with parallel.global_guidance (whose batch-wide normaliser 'clip' replaces)."""
        mode = getattr(self, "guidance_normaliser", "batch")
        if not isinstance(mode, str) or mode not in ("batch", "clip"):
            raise RohmB200Error(f"PoseNet: guidance_normaliser must be 'batch' or 'clip', got {mode!r}")
        if mode == "clip" and getattr(self, "guidance_sum_reducer", None) is not None:
            raise RohmB200Error("PoseNet: guidance_normaliser='clip' with parallel.global_guidance: the per-clip "
                                "normalisers need no collective and contradict the batch-wide one; disable one of them")
        return mode == "clip"

    def _lengths_on(self, values, device):
        """The per-clip lengths as an int32 device tensor (cached for the guided steps of one loop)."""
        cache = getattr(self, "_lengths_dev", None)
        if cache is None or cache[0] != values or cache[1] != device:
            cache = (values, device, torch.tensor(values, dtype=torch.int32, device=device))
            self._lengths_dev = cache
        return cache[2]

    def invalidate_cond(self):
        """Forget the cached step-invariant condition embedding (the samplers call this at the start of every loop,
        so a condition can never outlive the loop it was embedded for)."""
        if self._engine is not None:
            self._engine.cond_ref, self._engine.cond_version = None, -1

    # ---------------------------------------------------------------- test-time guidance
    def _norm_stats(self, device):
        key = (str(device), id(self.dataset))
        if getattr(self, "_norm_cache_key", None) != key:
            self._norm_cache = (torch.from_numpy(np.ascontiguousarray(self.dataset.Mean, dtype=np.float32)).to(device),
                                torch.from_numpy(np.ascontiguousarray(self.dataset.Std, dtype=np.float32)).to(device))
            self._norm_cache_key = key
        return self._norm_cache

    def guide_skating_with_smpl(self, batch, out, denoise_t, compute_grad='x_t'):
        """Gradient of -(foot-skating loss from SMPL-X joints + from the joint-based representation) w.r.t. x_t or the
        predicted x_0 (reference posenet.py:196-257), [bs, body_feat_dim, 1, T], trajectory and contact channels zero.
        One fused analytic forward+VJP (rohm_skating_guidance) instead of autograd through the body model; when nothing
        skates the result is an all-zero tensor (the reference returns a 0-dim zero), so no host sync is needed."""
        from .body_model import kernels_for
        x = batch['x_t'] if compute_grad == 'x_t' else out['pred_xstart']
        x = x.detach()
        x = x if (x.is_contiguous() and x.dtype == torch.float32) else x.contiguous().float()
        if self.dataset.traj_feat_dim != 22 or x.shape[1] != 294:
            raise RohmB200Error("guide_skating_with_smpl: implemented for the 294-channel representation with the "
                                "22-channel trajectory block (the configuration RoHM ships)")
        B, _, _, T = x.shape
        per_clip = self.guidance_per_clip()
        lengths = self.clip_lengths(batch, x.shape, grad_type='amass')
        mean, std = self._norm_stats(x.device)
        k = kernels_for(self.smplx_model, x.device, B * T, with_vertices=False)
        if per_clip:
            # each clip normalised by its own counts: clip b's gradient is that of clip b run alone
            lens = None if lengths is None else self._lengths_on(lengths, x.device)
            return k.skating_guidance(x, mean, std, lengths=lens, per_clip=True)
        if lengths is not None:
            # frames past a clip's length add nothing; the normalisers stay batch-wide over the real frames
            return k.skating_guidance(x, mean, std, lengths=self._lengths_on(lengths, x.device))
        reducer = getattr(self, "guidance_sum_reducer", None)
        if reducer is not None:
            # clip-sharded run reproducing the unsharded batch: the loss normalisers are batch-wide counts (reference
            # posenet.py:230-233), so the four sums are all-reduced over the ranks (rohm_b200.parallel.global_guidance)
            return k.skating_guidance_global(x, mean, std, reducer)
        return k.skating_guidance(x, mean, std)

    def _camera_affine(self, batch, device):
        """[B, 3, 4] canonical -> camera map of guide_2d_projection_with_smpl (reference posenet.py:285-297):
        p_cam = inv(cam_R) (inv(transf_matrix) p_cano - cam_t).  Per-clip 4x4 inverses: host-sized work, cached per
        transf_matrix tensor so the guided steps of one loop compute it once.

        With batch['cam2world'] [B,4,4] (windows.encode_video puts it there), clip b's camera is cam2world[b] instead of
        the dataset's cam_R / cam_t, so one batch can hold windows of recordings with different cameras.  A batch of one
        camera takes the dataset-camera path's operations (the same bits as that camera in the dataset); a batch of
        several computes each clip's affine as that clip alone would, so each clip gets the bits of its own run."""
        tm = batch['transf_matrix']
        c2w = batch.get('cam2world')
        c2w_version = None if c2w is None else c2w._version
        cache = getattr(self, "_cam_cache", None)
        if cache is not None and cache[0] is tm and cache[1] == tm._version and cache[2] is c2w and \
                cache[3] == c2w_version:
            return cache[4]
        cano2scene = torch.linalg.inv(tm.to(device=device, dtype=torch.float32))  # [B, 4, 4]

        def affine(cam_R, cam_t, c2s):
            Rinv = torch.linalg.inv(cam_R)
            M = Rinv @ c2s[:, 0:3, 0:3]                                       # [B, 3, 3]
            m = (Rinv @ (c2s[:, 0:3, 3] - cam_t).unsqueeze(-1))               # [B, 3, 1]
            return torch.cat([M, m], dim=-1)

        if c2w is None:
            cam_R = torch.as_tensor(self.dataset.cam_R, dtype=torch.float32, device=device).reshape(3, 3)
            cam_t = torch.as_tensor(self.dataset.cam_t, dtype=torch.float32, device=device).reshape(3)
            aff = affine(cam_R, cam_t, cano2scene).contiguous()
        else:
            B = cano2scene.shape[0]
            cams = c2w.to(device=device, dtype=torch.float32)
            if cams.shape != (B, 4, 4):
                raise RohmB200Error(f"guide_2d_projection_with_smpl: batch['cam2world'] must be [{B}, 4, 4], got "
                                    f"{tuple(cams.shape)}")
            # one camera (compared by bit pattern, so -0.0 and 0.0 differ; a host sync per new camera tensor, the affine
            # is cached for the loop's guided steps): the dataset-camera path's batched operations, and its bits
            rows16 = cams.reshape(B, 16).view(torch.int32).cpu()
            if bool((rows16 == rows16[0]).all()):
                aff = affine(cams[0, 0:3, 0:3], cams[0, 0:3, 3], cano2scene).contiguous()
            else:
                # several cameras: each clip by itself, with the operations and shapes of that clip run alone with its
                # camera as dataset.cam_R / cam_t (batched inverses and matrix products may round per batch size)
                tmd = tm.to(device=device, dtype=torch.float32)
                aff = torch.cat([affine(cams[b, 0:3, 0:3], cams[b, 0:3, 3], torch.linalg.inv(tmd[b:b + 1]))
                                 for b in range(B)]).contiguous()
        self._cam_cache = (tm, tm._version, c2w, c2w_version, aff)
        return aff

    def guide_2d_projection_with_smpl(self, batch, out, denoise_t, compute_grad='x_t'):
        """Gradient of -(2-D reprojection loss of 10 SMPL-X body joints against batch['keypoints_2d']) w.r.t. x_t or
        the predicted x_0 (reference posenet.py:260-317), [bs, body_feat_dim, 1, T], trajectory and contact channels
        zero.  One analytic forward + VJP kernel (rohm_projection_guidance) instead of autograd through the body model."""
        from .body_model import kernels_for
        x = batch['x_t'] if compute_grad == 'x_t' else out['pred_xstart']
        x = x.detach()
        x = x if (x.is_contiguous() and x.dtype == torch.float32) else x.contiguous().float()
        if self.dataset.traj_feat_dim != 22 or x.shape[1] != 294:
            raise RohmB200Error("guide_2d_projection_with_smpl: implemented for the 294-channel representation with the "
                                "22-channel trajectory block (the configuration RoHM ships)")
        B, _, _, T = x.shape
        per_clip = self.guidance_per_clip()
        lengths = self.clip_lengths(batch, x.shape, grad_type='prox')  # per-clip lengths need per-clip normalisers
        dev = x.device
        mean, std = self._norm_stats(dev)
        f32 = lambda t: t.to(device=dev, dtype=torch.float32).contiguous()
        kp = f32(batch['keypoints_2d'])
        if kp.dim() != 4 or kp.shape[0] != B or kp.shape[1] < T or kp.shape[2] != 22 or kp.shape[3] != 3:
            raise RohmB200Error(f"guide_2d_projection_with_smpl: batch['keypoints_2d'] must be [{B}, >={T}, 22, 3], got "
                                f"{tuple(kp.shape)}")
        k = kernels_for(self.smplx_model, dev, B * T, with_vertices=False)
        return k.projection_guidance(x, mean, std, self._camera_affine(batch, dev), f32(batch['focal_length']),
                                     f32(batch['camera_center']), kp, per_clip=per_clip,
                                     lengths=None if lengths is None else self._lengths_on(lengths, dev))

    def compute_losses_with_smpl(self, batch, model_output, smplx_model=None, epoch=0):
        """The evaluation loss dictionary of reference posenet.py:99-193 (what eval_losses returns with its default
        compute_loss=True, test_posenet.py:178); off the hot path, see rohm_b200/eval_losses.py."""
        from .eval_losses import posenet_losses
        return posenet_losses(self, batch, model_output, smplx_model, epoch)

    # ---------------------------------------------------------------- forward
    def forward(self, batch, timesteps):
        """batch['x_t'], batch['cond']: [bs, body_feat_dim, 1, T]; timesteps: [bs] int -> [bs, body_feat_dim, 1, T]
        (channels [0, traj_feat_dim) are batch['cond'][:, :traj_feat_dim], the rest is the denoised pose).
        batch['lengths'] (optional, integer [bs], 1 <= lengths[b] <= T): clip b has lengths[b] real frames; those come out
        bit-identical to running the clip alone, later frames come out zero and their inputs are never read."""
        e, x, ts = self.prepare(batch, timesteps)
        return e.forward(x, ts)

    def prepare(self, batch, timesteps):
        """forward up to the engine call: argument checks (host attribute reads), engine lookup and the step-invariant
        condition embedding (prepare_cond) -> (engine, x_t as a contiguous fp32 tensor, timesteps as contiguous int64)."""
        x_t, cond = batch['x_t'], batch['cond']
        if x_t.dim() != 4 or x_t.shape[2] != 1 or x_t.shape != cond.shape or x_t.shape[1] != self.input_feats:
            raise RohmB200Error(f"PoseNet: expected x_t/cond of shape [B, {self.input_feats}, 1, T], got "
                                f"{tuple(x_t.shape)} / {tuple(cond.shape)}")
        if timesteps.is_floating_point():
            # the reference indexes pe[timesteps]: a float index raises there too (rescale_timesteps is never enabled)
            raise RohmB200Error("PoseNet: timesteps must be an integer tensor (they index the positional table)")
        pe_rows = self.sequence_pos_encoder.pe.shape[0]
        if x_t.shape[3] + 1 > pe_rows:
            # T frames + the timestep token take T + 1 rows of the table; the reference's pe[:T + 1] add fails there too
            raise RohmB200Error(f"PoseNet: a clip of {x_t.shape[3]} frames needs {x_t.shape[3] + 1} rows of the positional "
                                f"table sequence_pos_encoder.pe, which has {pe_rows} (at most {pe_rows - 1} frames)")
        lengths = self.clip_lengths(batch, x_t.shape)
        e = self.prepare_cond(cond, lengths)
        x = x_t if (x_t.is_contiguous() and x_t.dtype == torch.float32) else x_t.contiguous().float()
        ts = timesteps.to(device=x.device, dtype=torch.int64).contiguous()
        return e, x, ts
