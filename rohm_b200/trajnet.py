"""TrajNet (1-D conv U-Net) and its TrajControl branch: drop-in for reference model/trajnet.py:10-275 (constructor,
attributes, state-dict keys, call signature) with the forward pass executed by the CUDA engine behind
``rohm_trajnet_*`` (include/rohm_b200.h).  The modules below only own parameters (see rohm_b200/heads.py).
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from ._lib import RohmB200Error
from .heads import Conv1dBlock, Downsample1d, ResidualTemporalBlock, SinusoidalPosEmb, Upsample1d, zero_module


class ControlNet(nn.Module):
    """TrajControl side branch: parameters only (keys ``controlnet.control_*``)."""

    def __init__(self, time_dim=32, control_cond_dim=272, traj_feat_dim=4, mid_dim=256):
        super().__init__()
        self.control_cond_dim = control_cond_dim
        self.traj_feat_dim = traj_feat_dim
        m = mid_dim
        rtb = lambda i, o: ResidualTemporalBlock(i, o, input_t=True, t_embed_dim=time_dim)
        self.control_zero_conv_0 = zero_module(nn.Conv1d(control_cond_dim, traj_feat_dim, 1, padding=0))
        self.control_enc1 = rtb(traj_feat_dim, m // 8)
        self.control_zero_conv_1 = zero_module(nn.Conv1d(m // 8, 32, 1, padding=0))
        self.control_downsample1 = Downsample1d(m // 8 * 2)
        self.control_enc2 = rtb(m // 8 * 2, m // 4)
        self.control_zero_conv_2 = zero_module(nn.Conv1d(m // 8 * 2, m // 8, 1, padding=0))
        self.control_downsample2 = Downsample1d(m // 4 * 2)
        self.control_enc3 = rtb(m // 4 * 2, m // 2)
        self.control_zero_conv_3 = zero_module(nn.Conv1d(m // 4 * 2, m // 4, 1, padding=0))
        self.control_downsample3 = Downsample1d(m // 2 * 2)
        self.control_enc4 = rtb(m // 2 * 2, m)
        self.control_zero_conv_4 = zero_module(nn.Conv1d(m, m // 4 * 2, 1, padding=0))
        self.control_downsample4 = Downsample1d(m * 2)
        self.control_mid_block1 = rtb(m * 2, m)
        self.control_mid_block2 = rtb(m, m)
        self.control_zero_conv_mid = zero_module(nn.Conv1d(m, m, 1, padding=0))

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("ControlNet is evaluated inside TrajNet's CUDA engine")


class TrajNet(nn.Module):
    def __init__(self, time_dim=32, cond_dim=4, mid_dim=256,
                 traj_feat_dim=4,
                 device=None, dataset=None,
                 repr_abs_only=False,
                 trajcontrol=False,
                 control_cond_dim=272,
                 weight_loss_root_rec_repr=0.0,
                 weight_loss_root_pos_global=0.0, weight_loss_root_vel_global=0.0,
                 weight_loss_root_rot_vel_from_abs_traj=0.0,
                 weight_loss_root_smplx_transl_vel=0.0, weight_loss_root_smplx_rot_vel=0.0,
                 weight_loss_root_smooth=0.0,
                 weight_loss_root_rot_cos_smooth_from_abs_traj=0.0,
                 ):
        super().__init__()
        self.traj_feat_dim = traj_feat_dim
        self.repr_abs_only = repr_abs_only
        self.time_dim, self.cond_dim, self.mid_dim = time_dim, cond_dim, mid_dim
        self.control_cond_dim = control_cond_dim
        self.trajcontrol = trajcontrol
        if self.trajcontrol:
            self.controlnet = ControlNet(time_dim=time_dim, control_cond_dim=control_cond_dim,
                                         traj_feat_dim=traj_feat_dim, mid_dim=mid_dim)
        self.weight_loss_root_rec_repr = weight_loss_root_rec_repr
        self.weight_loss_root_pos_global = weight_loss_root_pos_global
        self.weight_loss_root_vel_global = weight_loss_root_vel_global
        self.weight_loss_root_rot_vel_from_abs_traj = weight_loss_root_rot_vel_from_abs_traj
        self.weight_loss_root_smplx_transl_vel = weight_loss_root_smplx_transl_vel
        self.weight_loss_root_smplx_rot_vel = weight_loss_root_smplx_rot_vel
        self.weight_loss_root_smooth = weight_loss_root_smooth
        self.weight_loss_root_rot_cos_smooth_from_abs_traj = weight_loss_root_rot_cos_smooth_from_abs_traj
        self.dataset = dataset
        self.device = device
        m = mid_dim
        rtb = lambda i, o: ResidualTemporalBlock(i, o, input_t=True, t_embed_dim=time_dim)

        self.time_mlp = nn.Sequential(SinusoidalPosEmb(time_dim), nn.Linear(time_dim, time_dim * 4), nn.Mish(),
                                      nn.Linear(time_dim * 4, time_dim))
        # U-Net encoder
        self.diff_enc1 = rtb(self.traj_feat_dim, m // 8)
        self.diff_downsample1 = Downsample1d(m // 8 * 2)
        self.diff_enc2 = rtb(m // 8 * 2, m // 4)
        self.diff_downsample2 = Downsample1d(m // 4 * 2)
        self.diff_enc3 = rtb(m // 4 * 2, m // 2)
        self.diff_downsample3 = Downsample1d(m // 2 * 2)
        self.diff_enc4 = rtb(m // 2 * 2, m)
        self.diff_downsample4 = Downsample1d(m * 2)
        # middle
        self.diff_mid_block1 = rtb(m * 2, m)
        self.diff_mid_block2 = rtb(m, m)
        # decoder
        self.diff_upsample4 = Upsample1d(m)
        self.diff_dec4 = rtb(m * 2, m // 2)
        self.diff_upsample3 = Upsample1d(m // 2)
        self.diff_dec3 = rtb(m // 2 * 2, m // 4)
        self.diff_upsample2 = Upsample1d(m // 4)
        self.diff_dec2 = rtb(m // 4 * 2, m // 8)
        self.diff_upsample1 = Upsample1d(m // 8)
        self.diff_dec1 = rtb(m // 8 * 2, 32)
        self.diff_final_conv = nn.Sequential(Conv1dBlock(32, 32, kernel_size=5), nn.Conv1d(32, self.traj_feat_dim, 1))
        # condition pyramid (no time input)
        self.cond_enc1 = ResidualTemporalBlock(cond_dim, m // 8, input_t=False)
        self.cond_downsample1 = Downsample1d(m // 8)
        self.cond_enc2 = ResidualTemporalBlock(m // 8, m // 4, input_t=False)
        self.cond_downsample2 = Downsample1d(m // 4)
        self.cond_enc3 = ResidualTemporalBlock(m // 4, m // 2, input_t=False)
        self.cond_downsample3 = Downsample1d(m // 2)
        self.cond_enc4 = ResidualTemporalBlock(m // 2, m, input_t=False)
        self.cond_downsample4 = Downsample1d(m)  # present in checkpoints, never evaluated (reference :174)

        self.precision = None
        # True: the engine is created batch-invariant (rohm_trajnet_create_batch_invariant), so every real frame of a clip
        # depends on that clip alone, whatever B, padded T, position, engine or GPU.  A plain attribute: not in the state
        # dict, kept by .to() and load_state_dict.
        self.batch_invariant = False
        self._engine = None
        self._engine_fingerprint = None

    def invalidate_engine(self):
        self._engine = None

    def invalidate_cond(self):
        """Forget the cached condition pyramid (called by the samplers at the start of every loop)."""
        if self._engine is not None:
            self._engine.cond_ref, self._engine.control_ref = None, None

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._engine = None
        return super().load_state_dict(*a, **k)

    def compute_losses_with_smpl(self, batch, model_output, smplx_model=None):
        """The evaluation loss dictionary of reference trajnet.py:278-400 (what eval_losses returns with its default
        compute_loss=True, test_trajnet.py:154); off the hot path, see rohm_b200/eval_losses.py."""
        from .eval_losses import trajnet_losses
        return trajnet_losses(self, batch, model_output, smplx_model)

    def clip_lengths(self, batch, shape=None, grad_type=None):
        """batch['lengths'] checked against the padded [B, T, traj_dim] batch (`shape`, else batch['x_t'] / batch['cond']),
        as a tuple of ints; None when the key is absent.  Raises RohmB200Error before anything runs on the device.
        grad_type: accepted for the sampling loops' call; TrajNet has no guidance."""
        from .trajnet_engine import clip_lengths
        if shape is None and isinstance(batch, dict):
            shape = (batch['x_t'] if 'x_t' in batch else batch['cond']).shape
        return clip_lengths(batch, shape)

    def forward(self, batch, time):
        """batch['x_t'], batch['cond']: [bs, T, traj_dim]; batch['control_cond']: [bs, T, 272] when trajcontrol;
        time: [bs] int -> [bs, T, traj_dim] (reconstructed trajectory representation at timestep 0).
        batch['lengths'] (optional, integer [bs], multiples of 16 with 16 <= lengths[b] <= T): clip b has lengths[b] real
        frames; those depend on that clip alone, later frames come out zero and their inputs are never read."""
        e, x, ts = self.prepare(batch, time)
        return e.forward(x, ts)

    def prepare(self, batch, time):
        """trajnet_engine.prepare: -> (engine, x_t as a contiguous fp32 tensor, time as contiguous int64)."""
        from .trajnet_engine import prepare
        return prepare(self, batch, time)
