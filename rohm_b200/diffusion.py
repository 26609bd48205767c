"""Gaussian diffusion samplers for PoseNet and TrajNet on the CUDA engines.

API-compatible with the reference classes (diffusion/gaussian_diffusion_posenet.py ``GaussianDiffusionPoseNet``,
diffusion/gaussian_diffusion_trajnet.py ``GaussianDiffusionTrajNet``, diffusion/respace.py ``SpacedDiffusion*`` and
``_WrappedModel``): same constructor keywords, attributes (all float64 tables, ``num_timesteps``, ``timestep_map``),
method names, keyword arguments and return values.  What differs is where the work happens:

* the schedule is host numpy (rohm_b200.schedule), uploaded ONCE per device as an fp32 row table instead of four
  host->device table copies per step (reference ``_extract_into_tensor`` :967-980);
* the posterior mean, optional guidance terms and the noise injection are ONE fused kernel (rohm_ddpm_step) instead
  of ~10 elementwise launches (:212-234, :426-434, :461-479);
* the denoiser call goes to the CUDA engines (rohm_b200.posenet / rohm_b200.trajnet);
* the per-step ``t`` tensors and the respacing map live on the device for the whole loop (no per-step H2D).

Noise is drawn with ``torch.randn`` / ``torch.randn_like`` in exactly the reference's order (once for x_T, then once per
step including t == 0), so with the same seed on the same device the random stream is identical.  With
``batch['generators']`` (one CUDA generator per clip, rohm_b200.noise_streams) the same draws come from each clip's own
generator instead, as the clip alone would draw them.
"""
import enum
from copy import deepcopy

import numpy as np
import torch as th

from . import ops, schedule
from ._lib import RohmB200Error

import os

# ROHM_B200_FUSED_STEP=0: keep the explicit torch.randn_like + gather + update launches (developer / A-B switch)
_FUSED_STEP = os.environ.get("ROHM_B200_FUSED_STEP", "1") != "0"

get_named_beta_schedule = schedule.get_named_beta_schedule
betas_for_alpha_bar = schedule.betas_for_alpha_bar
space_timesteps = schedule.space_timesteps


class ModelMeanType(enum.Enum):
    PREVIOUS_X = enum.auto()
    START_X = enum.auto()
    EPSILON = enum.auto()


class ModelVarType(enum.Enum):
    LEARNED = enum.auto()
    FIXED_SMALL = enum.auto()
    FIXED_LARGE = enum.auto()
    LEARNED_RANGE = enum.auto()


class LossType(enum.Enum):
    MSE = enum.auto()
    RESCALED_MSE = enum.auto()
    KL = enum.auto()
    RESCALED_KL = enum.auto()

    def is_vb(self):
        return self == LossType.KL or self == LossType.RESCALED_KL


# Guidance schedule hard-coded by the reference (p_sample_with_grad, gaussian_diffusion_posenet.py:461-477), as
# (denoiser hook, weight, last respaced step index it applies on):
#   'amass': skating guidance, weight 3e6, on respaced step indices t <= 50
#   'prox' : 2-D reprojection guidance weight 3e5 then skating guidance weight 1e5, both on t <= 100
_GUIDANCE = {
    'amass': (('guide_skating_with_smpl', 3e6, 50),),
    'prox': (('guide_2d_projection_with_smpl', 3e5, 100), ('guide_skating_with_smpl', 1e5, 100)),
}


class _GaussianDiffusion:
    """Shared implementation; ``_POSENET`` selects the PoseNet-only features (guidance, early_stop)."""
    _POSENET = False

    def __init__(self, *, betas, model_mean_type, model_var_type, loss_type, rescale_timesteps=False, dataset=None,
                 device=''):
        self.model_mean_type = model_mean_type
        self.model_var_type = model_var_type
        self.loss_type = loss_type
        self.rescale_timesteps = rescale_timesteps
        self.dataset = dataset
        self.device = device
        tables = schedule.build_tables(betas)
        for name, arr in tables.items():
            setattr(self, name, arr)
        self.num_timesteps = int(self.betas.shape[0])
        self._coef_rows_host = schedule.ddpm_coef_rows(tables)
        self._dev_cache = {}
        # RNG entry points (kept as attributes so tests can inject a recorded noise stream)
        self._randn = th.randn
        self._randn_like = th.randn_like
        # (batch['generators'] list, NoiseStreams) of the sampling loop in progress, if it draws from per-clip streams
        self._loop_streams = None

    # ------------------------------------------------------------------ device-side tables
    def _dev(self, device):
        device = th.device(device)
        d = self._dev_cache.get(device)
        if d is None:
            d = {"coef": th.from_numpy(self._coef_rows_host).to(device), "tables": {}, "t_rows": {}}
            self._dev_cache[device] = d
        return d

    def _table(self, name, device):
        d = self._dev(device)["tables"]
        if name not in d:
            d[name] = th.from_numpy(np.ascontiguousarray(getattr(self, name))).to(device)
        return d[name]

    def _t_rows(self, batch_size, device):
        """int64 [num_timesteps, B] with row i == i: the per-step ``t`` tensors, built once instead of per step."""
        d = self._dev(device)["t_rows"]
        if batch_size not in d:
            d.clear()
            d[batch_size] = th.arange(self.num_timesteps, device=device, dtype=th.int64).unsqueeze(1).repeat(
                1, batch_size).contiguous()
        return d[batch_size]

    def _extract(self, name, t, broadcast_shape):
        res = self._table(name, t.device)[t].float()
        while len(res.shape) < len(broadcast_shape):
            res = res[..., None]
        return res.expand(broadcast_shape)

    def _coef_for(self, t):
        """fp32 [B, 8] coefficient rows {c1, c2, sigma, variance, ...} for a batch of step indices."""
        return self._dev(t.device)["coef"][t]

    # ------------------------------------------------------------------ q(.)
    def q_mean_variance(self, x_start, t):
        mean = self._extract("sqrt_alphas_cumprod", t, x_start.shape) * x_start
        variance = self._extract_expr(1.0 - self.alphas_cumprod, t, x_start.shape)
        log_variance = self._extract("log_one_minus_alphas_cumprod", t, x_start.shape)
        return mean, variance, log_variance

    def _extract_expr(self, arr, t, shape):
        res = th.from_numpy(np.ascontiguousarray(arr)).to(t.device)[t].float()
        while len(res.shape) < len(shape):
            res = res[..., None]
        return res.expand(shape)

    def q_sample(self, x_start, t, noise=None):
        """x_t ~ q(x_t | x_0) = sqrt(ac[t]) x_0 + sqrt(1 - ac[t]) noise."""
        if noise is None:
            noise = self._randn_like(x_start)
        assert noise.shape == x_start.shape
        B = x_start.shape[0]
        rows = th.zeros(B, 8, device=x_start.device, dtype=th.float32)
        rows[:, 0] = self._table("sqrt_alphas_cumprod", t.device)[t].float()
        rows[:, 2] = self._table("sqrt_one_minus_alphas_cumprod", t.device)[t].float()
        # same fused kernel: c1*x0 + 0*x0 + sigma*noise  (adding the exact zero product does not change the sum)
        xs = x_start.contiguous().float()
        return ops.ddpm_step(xs, xs, noise.contiguous().float(), rows)

    def q_posterior_mean_variance(self, x_start, x_t, t):
        assert x_start.shape == x_t.shape
        rows = self._coef_for(t).clone()
        rows[:, 2:] = 0
        xs = x_start.contiguous().float()
        mean = ops.ddpm_step(xs, x_t.contiguous().float(), xs, rows)
        var = self._extract("posterior_variance", t, x_t.shape)
        logvar = self._extract("posterior_log_variance_clipped", t, x_t.shape)
        assert mean.shape[0] == var.shape[0] == logvar.shape[0] == x_start.shape[0]
        return mean, var, logvar

    # ------------------------------------------------------------------ p(.)
    def p_mean_variance(self, model, batch, x, t, clip_denoised=True, denoised_fn=None, model_kwargs=None):
        """Runs the denoiser (x0-prediction, fixed-small variance; clip_denoised / denoised_fn are accepted and
        ignored exactly as in the reference) and returns {'mean','variance','log_variance','pred_xstart'}."""
        if model_kwargs is None:
            model_kwargs = {}
        B = x.shape[0]
        assert t.shape == (B,)
        batch['x_t'] = x
        pred_xstart = model(batch, self._scale_timesteps(t), **model_kwargs)
        mean, var, logvar = self.q_posterior_mean_variance(x_start=pred_xstart, x_t=x, t=t)
        return {"mean": mean, "variance": var, "log_variance": logvar, "pred_xstart": pred_xstart}

    def _predict_xstart_from_eps(self, x_t, t, eps):
        assert x_t.shape == eps.shape
        return (self._extract("sqrt_recip_alphas_cumprod", t, x_t.shape) * x_t
                - self._extract("sqrt_recipm1_alphas_cumprod", t, x_t.shape) * eps)

    def _predict_xstart_from_xprev(self, x_t, t, xprev):
        assert x_t.shape == xprev.shape
        return (self._extract_expr(1.0 / self.posterior_mean_coef1, t, x_t.shape) * xprev
                - self._extract_expr(self.posterior_mean_coef2 / self.posterior_mean_coef1, t, x_t.shape) * x_t)

    def _predict_eps_from_xstart(self, x_t, t, pred_xstart):
        return (self._extract("sqrt_recip_alphas_cumprod", t, x_t.shape) * x_t - pred_xstart) / \
            self._extract("sqrt_recipm1_alphas_cumprod", t, x_t.shape)

    def _scale_timesteps(self, t):
        if self.rescale_timesteps:
            return t.float() * (1000.0 / self.num_timesteps)
        return t

    def condition_mean(self, cond_fn, p_mean_var, x, t, model_kwargs=None):
        gradient = cond_fn(x, self._scale_timesteps(t), **(model_kwargs or {}))
        return p_mean_var["mean"].float() + p_mean_var["variance"] * gradient.float()

    def condition_mean_with_grad(self, cond_fn, p_mean_var, x, t, model_kwargs=None):
        gradient = cond_fn(x, t, p_mean_var, **(model_kwargs or {}))
        return p_mean_var["mean"].float() + p_mean_var["variance"] * gradient.float()

    def condition_score(self, cond_fn, p_mean_var, x, t, model_kwargs=None):
        alpha_bar = self._extract("alphas_cumprod", t, x.shape)
        eps = self._predict_eps_from_xstart(x, t, p_mean_var["pred_xstart"])
        eps = eps - (1 - alpha_bar).sqrt() * cond_fn(x, self._scale_timesteps(t), **(model_kwargs or {}))
        out = p_mean_var.copy()
        out["pred_xstart"] = self._predict_xstart_from_eps(x, t, eps)
        out["mean"], _, _ = self.q_posterior_mean_variance(x_start=out["pred_xstart"], x_t=x, t=t)
        return out

    def condition_score_with_grad(self, cond_fn, p_mean_var, x, t, model_kwargs=None):
        alpha_bar = self._extract("alphas_cumprod", t, x.shape)
        eps = self._predict_eps_from_xstart(x, t, p_mean_var["pred_xstart"])
        eps = eps - (1 - alpha_bar).sqrt() * cond_fn(x, t, p_mean_var, **(model_kwargs or {}))
        out = p_mean_var.copy()
        out["pred_xstart"] = self._predict_xstart_from_eps(x, t, eps)
        out["mean"], _, _ = self.q_posterior_mean_variance(x_start=out["pred_xstart"], x_t=x, t=t)
        return out

    # ------------------------------------------------------------------ one ancestral step
    def _denoise(self, model, batch, x, t, model_kwargs):
        B = x.shape[0]
        assert t.shape == (B,)
        if x.device.type != "cuda":
            raise RohmB200Error("rohm_b200 diffusion: tensors must live on a CUDA device (there is no CPU path)")
        x = x if (x.is_contiguous() and x.dtype == th.float32) else x.contiguous().float()
        batch['x_t'] = x
        return x, model(batch, self._scale_timesteps(t), **(model_kwargs or {}))

    def _wrap_model(self, model):
        return model  # the respaced subclasses wrap the denoiser so that it sees original timesteps

    def _noise_in_kernel(self, x):
        """The noise may be drawn inside the update kernel when it comes from torch's own CUDA generator (bit-identical
        stream, see ops.ddpm_step_philox); an injected noise source (tests, sharded parity noise) keeps the explicit tensor."""
        return self._randn_like is th.randn_like and x.is_cuda and _FUSED_STEP

    # ------------------------------------------------------------------ per-clip noise streams (batch['generators'])
    def _channels_last(self):
        return not self._POSENET  # PoseNet batches are [B, C, 1, T], TrajNet batches [B, T, C]

    def _draw_lengths(self, model, batch, shape):
        """The per-clip lengths the draws of a [B, ...] batch follow (the denoiser's check of batch['lengths']), or None."""
        if batch.get('lengths') is None:
            return None
        return _inner(model).clip_lengths(batch, shape)

    def _open_streams(self, batch, shape, device, const_noise=False):
        """NoiseStreams of batch['generators'] after the validator's checks, or None without the key."""
        from .noise_streams import NoiseStreams, check_generators
        gens = check_generators(batch, shape[0], device, diffusion=self, const_noise=const_noise)
        return None if gens is None else NoiseStreams(gens, device)

    def _step_streams(self, batch, x, const_noise=False):
        """(streams, owned) of one step: the loop's streams when the step runs inside a loop over this batch's generators,
        else streams opened for this call alone (owned: the caller closes them, writing the offsets back)."""
        if not isinstance(batch, dict) or batch.get('generators') is None:
            return None, False
        ls = self._loop_streams
        if ls is not None and ls[0] is batch['generators']:
            return ls[1], False
        return self._open_streams(batch, x.shape, x.device, const_noise), True

    def _draw_noise(self, model, batch, x, streams):
        """An explicit noise tensor like x: each clip's draw from its stream, else self._randn_like."""
        if streams is None:
            return self._randn_like(x)
        return ops.randn_clips(streams, x.shape, self._channels_last(), self._draw_lengths(model, batch, x.shape),
                               device=x.device)

    def _coef_row(self, t, step_index):
        """The step's coefficient row: a view of the per-device table when the (batch-uniform) step index is known to the
        host, else a gather by the per-clip indices."""
        if step_index is not None:
            return self._dev(t.device)["coef"][int(step_index)]
        return self._coef_for(t)

    # ------------------------------------------------------------------ one ancestral step
    def _step(self, model, batch, x, t, step_index, streams, terms=(), cond_fn=None, const_noise=False,
              model_kwargs=None):
        """x_{t-1} = coef1[t] x0 + coef2[t] x_t (+ guidance) + (t != 0) exp(0.5 logvar[t]) noise, x0 = model(batch | x_t, t)
        -> {'sample', 'pred_xstart', 'x_t'}.  Decides, in this order:

        1. the fused step: the denoiser's forward and the update as ONE graph launch (engine.sample_step), when there are
           no guidance terms, no cond_fn, no const_noise and no model kwargs, the step index is known to the host, the
           noise is drawn in the kernel (_noise_in_kernel), t holds integer step indices that are not rescaled, and the
           denoiser has prepare().  The same arithmetic and the same noise as the separate launches below;
        2. otherwise the denoiser call, then the noise: drawn inside the update kernel from torch's generator or from the
           per-clip streams, or an explicit tensor when the noise source is replaced, _FUSED_STEP is off, const_noise is
           on (clip 0's noise for every clip) or a cond_fn is given;
        3. guidance: `terms` are (hook, weight) pairs; hook k's gradient w.r.t. pred_xstart enters the update scaled by
           the fp32 product weight * variance[t] (coefficient column 3 + k), as the reference forms it.  A 0-dim gradient
           ("nothing skates") adds nothing;
        4. one update launch.  A TrajNet cond_fn instead shifts the posterior mean by condition_mean (reference
           gaussian_diffusion_trajnet.py:433-436); a PoseNet cond_fn is not applied, as in the reference's p_sample."""
        if (not terms and cond_fn is None and not const_noise and not model_kwargs and step_index is not None and
                self._noise_in_kernel(x) and not t.is_floating_point() and not self.rescale_timesteps):
            wrapped = self._wrap_model(model)  # respaced schedules: step index -> original timestep
            prepare = getattr(_inner(wrapped), "prepare", None)
            if prepare is not None:
                batch['x_t'] = x
                e, x, ts = prepare(batch, wrapped.map_timesteps(t) if isinstance(wrapped, _WrappedModel) else t)
                batch['x_t'] = x
                x0, nxt = e.sample_step(x, ts, self._coef_row(t, step_index), streams=streams)
                return {"sample": nxt, "pred_xstart": x0, "x_t": x}
        x, x0 = self._denoise(model, batch, x, t, model_kwargs)
        noise = None
        if const_noise or cond_fn is not None or not self._noise_in_kernel(x):
            noise = self._draw_noise(model, batch, x, streams)
            if const_noise:
                noise = noise[[0]].repeat(x.shape[0], *([1] * (x.dim() - 1)))
        if cond_fn is not None and not self._POSENET:
            mean, var, logvar = self.q_posterior_mean_variance(x0, x, t)
            out = {"mean": mean, "variance": var, "log_variance": logvar, "pred_xstart": x0}
            mean = self.condition_mean(cond_fn, out, x, t, model_kwargs=model_kwargs)
            nonzero = (t != 0).float().view(-1, *([1] * (x.dim() - 1)))
            sample = mean + nonzero * th.exp(0.5 * logvar) * noise
            return {"sample": sample, "pred_xstart": x0, "x_t": x}
        coef = self._coef_row(t, step_index)
        grads, scales = [], []
        for hook, weight in terms:
            g = hook(batch, {"pred_xstart": x0}, t, compute_grad='x_0')
            if g.dim() != 0:
                grads.append(g.contiguous().float())
                scales.append(weight)
        if grads:
            coef = coef.expand(x.shape[0], -1) if coef.dim() == 1 else coef
            var = coef[:, 3].clone()
            coef = coef.clone()
            for k, w in enumerate(scales):
                coef[:, 3 + k] = w * var  # fp32 product weight * variance[t], as the reference forms it
        grads = tuple(grads)
        if noise is not None:
            sample = ops.ddpm_step(x0, x, noise, coef, grads=grads)
        elif streams is not None:
            sample = ops.ddpm_step_philox_clips(x0, x, coef, streams, self._channels_last(),
                                                self._draw_lengths(model, batch, x.shape), grads=grads)
        else:
            sample = ops.ddpm_step_philox(x0, x, coef, grads=grads)
        return {"sample": sample, "pred_xstart": x0, "x_t": x}

    def p_sample(self, model, batch, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None,
                 const_noise=False, _step_index=None):
        """x_{t-1} = coef1[t] x0 + coef2[t] x_t + (t != 0) exp(0.5 logvar[t]) noise, x0 = model(batch | x_t, t).
        Returns {'sample', 'pred_xstart', 'x_t'}.  With batch['generators'] clip b's noise comes from generators[b]
        (rohm_b200.noise_streams)."""
        streams, owned = self._step_streams(batch, x, const_noise)
        try:
            return self._step(model, batch, x, t, _step_index, streams, cond_fn=cond_fn, const_noise=const_noise,
                              model_kwargs=model_kwargs)
        finally:
            if owned:
                streams.close()

    def p_sample_with_grad(self, model, batch, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None, grad_type=None,
                           model_kwargs=None, const_noise=False, _step_index=None):
        """PoseNet: p_sample plus the hard-coded test-time guidance schedule _GUIDANCE[grad_type] (an unknown grad_type
        applies none, as in the reference); TrajNet: p_sample without guidance.  The update ignores cond_fn and
        const_noise, as the reference's does; const_noise with batch['generators'] is still refused."""
        streams, owned = self._step_streams(batch, x, const_noise)
        try:
            terms = ()
            if grad_type in _GUIDANCE:
                step = int(t[0]) if _step_index is None else int(_step_index)  # the reference syncs on t[0] every step
                terms = [(getattr(model, hook), weight) for hook, weight, last in _GUIDANCE[grad_type] if step <= last]
            return self._step(model, batch, x, t, _step_index, streams, terms, model_kwargs=model_kwargs)
        finally:
            if owned:
                streams.close()

    # ------------------------------------------------------------------ loops
    def _begin_loop(self, model, grad_type=None, batch=None, shape=None, device=None, const_noise=False):
        """Once per sampling loop, before any step: drop the denoiser's cached step-invariant condition embedding (a
        condition tensor can never outlive the loop it was embedded for) and reject what cannot run BEFORE a thousand
        denoiser steps are spent (the reference would fail, or silently do nothing, at the first guided step), per-clip
        lengths and generators included.  Returns the loop's NoiseStreams with batch['generators'] (the caller closes
        them when the loop ends), else None."""
        inner = _inner(model)
        if grad_type is not None and self._POSENET and hasattr(inner, "guidance_per_clip"):
            inner.guidance_per_clip()  # a bad guidance_normaliser, or 'clip' with global_guidance
        if not self._POSENET and hasattr(inner, "batch_invariant"):
            from .trajnet_engine import batch_invariant
            batch_invariant(inner)  # a non-bool TrajNet.batch_invariant
        if batch is not None and batch.get('lengths') is not None and hasattr(inner, "clip_lengths"):
            inner.clip_lengths(batch, shape, grad_type=grad_type)
        streams = None
        if batch is not None and batch.get('generators') is not None:
            from .noise_streams import check_generators
            check_generators(batch, shape[0], device, diffusion=self, const_noise=const_noise)
        inv = getattr(inner, "invalidate_cond", None)
        if inv is not None:
            inv()
        if grad_type is not None and self._POSENET and grad_type in _GUIDANCE:
            for hook, _, _ in _GUIDANCE[grad_type]:
                if not hasattr(inner, hook):
                    raise RohmB200Error(f"grad_type={grad_type!r} needs model.{hook}")
        tmap = getattr(self, "timestep_map", None)
        pe = getattr(getattr(inner, "sequence_pos_encoder", None), "pe", None)
        if tmap is not None and pe is not None and len(tmap) and max(tmap) >= pe.shape[0]:
            raise RohmB200Error(f"timestep {max(tmap)} exceeds the positional table ({pe.shape[0]} rows) that embeds it")
        if batch is not None and batch.get('generators') is not None:
            streams = self._open_streams(batch, shape, device, const_noise)
        if streams is not None:
            self._loop_streams = (batch['generators'], streams)
        return streams

    def _end_loop(self, streams):
        """When a loop returns or its generator is closed: writes the generators' offsets back."""
        if streams is None:
            return
        if self._loop_streams is not None and self._loop_streams[1] is streams:
            self._loop_streams = None
        streams.close()

    def _initial_noise(self, model, batch, shape, device, noise, streams):
        """x_T: the caller's `noise`, else per-clip streams, else the global generator."""
        if noise is not None:
            return noise
        if streams is not None:
            return ops.randn_clips(streams, shape, self._channels_last(), self._draw_lengths(model, batch, shape),
                                   device=device)
        return self._randn(*shape, device=device)

    def _loop(self, model, batch, shape, noise, device, progress, skip_timesteps, init_image, step, grad_type=None,
              const_noise=False, early_stop=False):
        """The loop structure the ancestral and DDIM samplers share: x_T (or init_image noised to the first step), then
        step(x, t, i) -> out from i = T-1 - skip_timesteps down to 0 (the first 980 steps with early_stop), yielding each
        out and continuing from out['sample']."""
        if device is None:
            device = next(model.parameters()).device
        assert isinstance(shape, (tuple, list))
        streams = self._begin_loop(model, grad_type, batch, shape, device, const_noise)
        try:
            img = self._initial_noise(model, batch, shape, device, noise, streams)
            if skip_timesteps and init_image is None:
                init_image = th.zeros_like(img)
            indices = list(range(self.num_timesteps - skip_timesteps))[::-1]
            t_rows = self._t_rows(shape[0], device)
            if init_image is not None:
                img = self.q_sample(init_image, t_rows[indices[0]], img)
            if early_stop:
                indices = indices[0:980]
            if progress:
                from tqdm.auto import tqdm
                indices = tqdm(indices)
            for i in indices:
                with th.no_grad():
                    out = step(img, t_rows[i], i)
                    yield out
                    img = out["sample"]
        finally:
            self._end_loop(streams)

    def p_sample_loop(self, model, batch, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                      model_kwargs=None, device=None, progress=False, skip_timesteps=0, init_image=None,
                      randomize_class=False, cond_fn_with_grad=False, grad_type=None, early_stop=False, dump_steps=None,
                      const_noise=False, save_intermediate_result=False):
        """Runs the whole chain; returns the final sample (``pred_xstart`` of the last executed step if
        ``early_stop``), or the dumps / intermediate lists in the two diagnostic modes of the reference."""
        if (grad_type is not None or early_stop) and not self._POSENET:
            raise TypeError("grad_type / early_stop are PoseNet-only arguments")
        final = None
        dump = [] if dump_steps is not None else None
        inter_x0, inter_xt, inter_t = [], [], []
        i = -1
        for i, sample in enumerate(self.p_sample_loop_progressive(
                model, batch, shape, noise=noise, clip_denoised=clip_denoised, denoised_fn=denoised_fn, cond_fn=cond_fn,
                model_kwargs=model_kwargs, device=device, progress=progress, skip_timesteps=skip_timesteps,
                init_image=init_image, randomize_class=randomize_class, cond_fn_with_grad=cond_fn_with_grad,
                grad_type=grad_type, early_stop=early_stop, const_noise=const_noise)):
            if dump is not None and i in dump_steps:
                dump.append(deepcopy(sample["sample"]))
            final = sample
            if save_intermediate_result and i % (self.num_timesteps // 5) == 0:
                inter_x0.append(sample['pred_xstart'].clone().detach())
                inter_xt.append(sample['x_t'].clone().detach())
                inter_t.append(self.num_timesteps - i - 1)
        if dump is not None:
            return dump
        if not save_intermediate_result:
            return final["pred_xstart"] if early_stop else final["sample"]
        inter_x0.append(final['pred_xstart'].clone().detach())
        inter_xt.append(final['x_t'].clone().detach())
        inter_t.append(self.num_timesteps - i - 1)
        return final['sample'], inter_x0, inter_xt, inter_t

    def p_sample_loop_progressive(self, model, batch, shape, noise=None, clip_denoised=True, denoised_fn=None,
                                  cond_fn=None, model_kwargs=None, device=None, progress=False, skip_timesteps=0,
                                  init_image=None, randomize_class=False, cond_fn_with_grad=False, grad_type=None,
                                  early_stop=False, const_noise=False):
        """Generator over the per-step dicts, from t = T-1 down to 0 (or the first 980 steps with early_stop)."""
        sample_fn = self.p_sample_with_grad if cond_fn_with_grad else self.p_sample
        kw = dict(grad_type=grad_type) if cond_fn_with_grad and self._POSENET else {}
        yield from self._loop(
            model, batch, shape, noise, device, progress, skip_timesteps, init_image,
            lambda x, t, i: sample_fn(model, batch, x, t, clip_denoised=clip_denoised, denoised_fn=denoised_fn,
                                      cond_fn=cond_fn, model_kwargs=model_kwargs, const_noise=const_noise,
                                      _step_index=i, **kw),
            grad_type if cond_fn_with_grad else None, const_noise, early_stop)

    # ------------------------------------------------------------------ DDIM
    # The reference's ddim_* methods cannot run (they call p_mean_variance without `batch`, and eval_losses never
    # reaches them -- SURVEY.md D4).  These implement the update those methods spell out, with `batch` threaded.
    def ddim_sample(self, model, batch, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None, model_kwargs=None,
                    eta=0.0, _step_index=None):
        if cond_fn is not None:
            raise NotImplementedError("cond_fn with DDIM sampling (condition_score) is not on the supported path")
        streams, owned = self._step_streams(batch, x)
        try:
            x, x0 = self._denoise(model, batch, x, t, model_kwargs)
            noise = self._draw_noise(model, batch, x, streams)
        finally:
            if owned:
                streams.close()
        step = int(t[0]) if _step_index is None else _step_index
        sample = ops.ddim_step(x0, x, noise, schedule.ddim_coefs(self.__dict__, step, eta))
        return {"sample": sample, "pred_xstart": x0}

    def ddim_sample_loop(self, model, batch, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                         model_kwargs=None, device=None, progress=False, eta=0.0, skip_timesteps=0, init_image=None,
                         randomize_class=False, cond_fn_with_grad=False, dump_steps=None, const_noise=False):
        if dump_steps is not None or const_noise:
            raise NotImplementedError()
        if cond_fn_with_grad:
            raise RohmB200Error("ddim_sample_loop: test-time guidance (cond_fn_with_grad / grad_type) is defined for the "
                                "ancestral sampler only (the reference's ddim_sample_with_grad cannot run, SURVEY D4); "
                                "use a non-'ddim' respacing or cond_fn_with_grad=False")
        final = None
        for sample in self.ddim_sample_loop_progressive(
                model, batch, shape, noise=noise, clip_denoised=clip_denoised, denoised_fn=denoised_fn, cond_fn=cond_fn,
                model_kwargs=model_kwargs, device=device, progress=progress, eta=eta, skip_timesteps=skip_timesteps,
                init_image=init_image):
            final = sample
        return final["sample"]

    def ddim_sample_loop_progressive(self, model, batch, shape, noise=None, clip_denoised=True, denoised_fn=None,
                                     cond_fn=None, model_kwargs=None, device=None, progress=False, eta=0.0,
                                     skip_timesteps=0, init_image=None, randomize_class=False, cond_fn_with_grad=False):
        yield from self._loop(
            model, batch, shape, noise, device, progress, skip_timesteps, init_image,
            lambda x, t, i: self.ddim_sample(model, batch, x, t, clip_denoised=clip_denoised, denoised_fn=denoised_fn,
                                             cond_fn=cond_fn, model_kwargs=model_kwargs, eta=eta, _step_index=i))

    # ------------------------------------------------------------------ entry points used by the drivers
    def training_losses(self, *a, **k):
        raise NotImplementedError("rohm_b200 implements the inference hot path; training losses are out of scope "
                                  "(see DESIGN.md)")

    def _sample_for_eval(self, model, batch, shape, progress, clip_denoised, cond_fn_with_grad, timestep_respacing,
                         grad_type=None, early_stop=False):
        inner = _inner(model)
        if isinstance(timestep_respacing, str) and timestep_respacing.startswith('ddim'):
            # the branch the reference left commented out (:949-952); it has no guidance / early-stop variant, so asking
            # for them is an error rather than a silently unguided run
            if early_stop or (cond_fn_with_grad and grad_type is not None):
                raise RohmB200Error("eval_losses(timestep_respacing='ddim...'): grad_type / early_stop are only defined "
                                    "for the ancestral sampler; drop them or use a non-'ddim' respacing")
            return self.ddim_sample_loop(model=inner, batch=batch, shape=shape, progress=progress,
                                         clip_denoised=clip_denoised, eta=0.0)
        kw = dict(grad_type=grad_type, early_stop=early_stop) if self._POSENET else {}
        return self.p_sample_loop(model=inner, batch=batch, shape=shape, progress=progress, clip_denoised=clip_denoised,
                                  cond_fn_with_grad=cond_fn_with_grad, **kw)


def _refuse_losses_with_lengths(batch, compute_loss):
    if compute_loss and batch.get('lengths') is not None:
        raise RohmB200Error("eval_losses: the loss dictionary over clips with batch['lengths'] is out of scope (it "
                            "would average over padded frames); pass compute_loss=False and score each clip's frames")


class GaussianDiffusionPoseNet(_GaussianDiffusion):
    _POSENET = True

    def eval_losses(self, model, batch, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                    device=None, progress=False, skip_timesteps=0, init_data=None, randomize_class=False,
                    cond_fn_with_grad=False, grad_type=None, early_stop=False, cond_grad_weight=1.0, dump_steps=None,
                    const_noise=False, cur_epoch=0, timestep_respacing='', compute_loss=True, smplx_model=None, epoch=0):
        """The call the drivers make (test_amass_full.py:376, test_posenet.py:178): full sampling loop, then the
        optional loss dict.  Returns (loss_dict | None, model_output)."""
        _refuse_losses_with_lengths(batch, compute_loss)
        model_output = self._sample_for_eval(model, batch, shape, progress, clip_denoised, cond_fn_with_grad,
                                             timestep_respacing, grad_type=grad_type, early_stop=early_stop)
        inner = _inner(model)
        loss_dict = inner.compute_losses_with_smpl(batch, model_output, smplx_model, epoch) if compute_loss else None
        return loss_dict, model_output


class GaussianDiffusionTrajNet(_GaussianDiffusion):
    _POSENET = False

    def p_sample_with_grad(self, model, batch, x, t, clip_denoised=True, denoised_fn=None, cond_fn=None,
                           model_kwargs=None, const_noise=False, _step_index=None):
        return super().p_sample_with_grad(model, batch, x, t, clip_denoised=clip_denoised, denoised_fn=denoised_fn,
                                          cond_fn=cond_fn, grad_type=None, model_kwargs=model_kwargs,
                                          _step_index=_step_index)

    def p_sample_loop(self, model, batch, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                      model_kwargs=None, device=None, progress=False, skip_timesteps=0, init_image=None,
                      randomize_class=False, cond_fn_with_grad=False, dump_steps=None, const_noise=False,
                      save_intermediate_result=False):
        return super().p_sample_loop(model, batch, shape, noise=noise, clip_denoised=clip_denoised,
                                     denoised_fn=denoised_fn, cond_fn=cond_fn, model_kwargs=model_kwargs, device=device,
                                     progress=progress, skip_timesteps=skip_timesteps, init_image=init_image,
                                     randomize_class=randomize_class, cond_fn_with_grad=cond_fn_with_grad,
                                     dump_steps=dump_steps, const_noise=const_noise,
                                     save_intermediate_result=save_intermediate_result)

    def eval_losses(self, model, batch, shape, noise=None, clip_denoised=True, denoised_fn=None, cond_fn=None,
                    device=None, progress=False, skip_timesteps=0, init_data=None, randomize_class=False,
                    cond_fn_with_grad=False, cond_grad_weight=1.0, dump_steps=None, const_noise=False, cur_epoch=0,
                    timestep_respacing='', compute_loss=True, smplx_model=None):
        """test_amass_full.py:245/259, test_trajnet.py:154.  Returns (loss_dict | None, model_output)."""
        _refuse_losses_with_lengths(batch, compute_loss)
        model_output = self._sample_for_eval(model, batch, shape, progress, clip_denoised, cond_fn_with_grad,
                                             timestep_respacing)
        inner = _inner(model)
        loss_dict = inner.compute_losses_with_smpl(batch, model_output, smplx_model) if compute_loss else None
        return loss_dict, model_output


# ---------------------------------------------------------------------------------------------------------------
# respacing
# ---------------------------------------------------------------------------------------------------------------
class _WrappedModel:
    """Maps the respaced step index to the original timestep before calling the denoiser (respace.py:183-195).
    The map lives on the device once instead of being rebuilt from a python list on every call."""

    def __init__(self, model, timestep_map, rescale_timesteps, original_num_steps):
        self.model = model
        self.timestep_map = timestep_map
        self.rescale_timesteps = rescale_timesteps
        self.original_num_steps = original_num_steps
        self._maps = {}

    def parameters(self):
        return self.model.parameters()

    def _map(self, ts):
        key = (ts.device, ts.dtype)
        m = self._maps.get(key)
        if m is None:
            m = th.tensor(self.timestep_map, device=ts.device, dtype=ts.dtype)
            self._maps[key] = m
        return m

    def map_timesteps(self, ts):
        """Original timesteps of a batch of step indices (what __call__ hands to the denoiser); the identity map of an
        un-respaced schedule needs no gather."""
        if self.timestep_map == list(range(len(self.timestep_map))):
            return ts
        return self._map(ts)[ts]

    def __call__(self, x, ts, **kwargs):
        new_ts = self.map_timesteps(ts)
        if self.rescale_timesteps:
            new_ts = new_ts.float() * (1000.0 / self.original_num_steps)
        return self.model(x, new_ts, **kwargs)

    def __getattr__(self, name):
        # guidance hooks (guide_skating_with_smpl, ...) are looked up on the wrapped denoiser
        return getattr(self.__dict__["model"], name)


def _inner(model):
    """The denoiser behind a respacing wrapper."""
    return model.model if isinstance(model, _WrappedModel) else model


def _spaced(base_cls):
    class Spaced(base_cls):
        def __init__(self, use_timesteps, **kwargs):
            self.use_timesteps = set(use_timesteps)
            self.original_num_steps = len(kwargs["betas"])
            new_betas, self.timestep_map = schedule.respace(kwargs["betas"], self.use_timesteps)
            kwargs["betas"] = new_betas
            super().__init__(**kwargs)
            self._wrapped = {}

        def _wrap_model(self, model):
            if isinstance(model, _WrappedModel):
                return model
            w = self._wrapped.get(id(model))
            if w is None or w.model is not model:
                w = _WrappedModel(model, self.timestep_map, self.rescale_timesteps, self.original_num_steps)
                self._wrapped = {id(model): w}
            return w

        def p_mean_variance(self, model, *args, **kwargs):
            return super().p_mean_variance(self._wrap_model(model), *args, **kwargs)

        def _denoise(self, model, *args, **kwargs):
            return super()._denoise(self._wrap_model(model), *args, **kwargs)

        def training_losses(self, model, *args, **kwargs):
            return super().training_losses(self._wrap_model(model), *args, **kwargs)

        def eval_losses(self, model, *args, **kwargs):
            return super().eval_losses(self._wrap_model(model), *args, **kwargs)

        def condition_mean(self, cond_fn, *args, **kwargs):
            return super().condition_mean(self._wrap_model(cond_fn), *args, **kwargs)

        def condition_score(self, cond_fn, *args, **kwargs):
            return super().condition_score(self._wrap_model(cond_fn), *args, **kwargs)

        def _scale_timesteps(self, t):
            return t  # scaling is done by the wrapped model

    return Spaced


SpacedDiffusionPoseNet = _spaced(GaussianDiffusionPoseNet)
SpacedDiffusionPoseNet.__name__ = SpacedDiffusionPoseNet.__qualname__ = "SpacedDiffusionPoseNet"
SpacedDiffusionTrajNet = _spaced(GaussianDiffusionTrajNet)
SpacedDiffusionTrajNet.__name__ = SpacedDiffusionTrajNet.__qualname__ = "SpacedDiffusionTrajNet"


def create_gaussian_diffusion(args, gd, return_class, num_diffusion_timesteps=100, timestep_respacing='', device='',
                              dataset=None):
    """utils/model_util.py:6-40.  ``gd`` is the diffusion *module* (it must expose get_named_beta_schedule, LossType,
    ModelMeanType, ModelVarType); x0-prediction, fixed variance, no timestep rescaling, MSE loss."""
    steps = num_diffusion_timesteps
    betas = gd.get_named_beta_schedule(args.noise_schedule, steps, 1.)
    if not timestep_respacing:
        timestep_respacing = [steps]
    return return_class(
        use_timesteps=space_timesteps(steps, timestep_respacing),
        betas=betas,
        model_mean_type=gd.ModelMeanType.START_X,
        model_var_type=(gd.ModelVarType.FIXED_LARGE if not args.sigma_small else gd.ModelVarType.FIXED_SMALL),
        loss_type=gd.LossType.MSE,
        rescale_timesteps=False,
        dataset=dataset,
        device=device,
    )
