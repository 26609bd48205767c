"""Host-side clip-length check of PoseNet.forward (no GPU needed): T frames plus the timestep token must fit in the
positional table, as in the reference, and the check fires before any engine is built."""
import pytest
import torch

from rohm_b200 import synthetic
from rohm_b200._lib import RohmB200Error
from rohm_b200.posenet import PoseNet


def _model():
    ds = synthetic.make_dataset('pose')
    return PoseNet(dataset=ds, body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4, device=None,
                   traj_feat_dim=22).eval()


def test_clip_longer_than_the_positional_table_is_refused_before_the_engine():
    m = _model()
    rows = m.sequence_pos_encoder.pe.shape[0]
    x = torch.zeros(1, 294, 1, rows)
    with pytest.raises(RohmB200Error, match=r"sequence_pos_encoder\.pe"):
        m({'x_t': x, 'cond': x}, torch.tensor([3]))
    assert m._engine is None
    # one frame less passes the check and reaches the device requirement (CPU tensors are refused there)
    x = torch.zeros(1, 294, 1, rows - 1)
    with pytest.raises(RohmB200Error, match="CUDA device"):
        m({'x_t': x, 'cond': x}, torch.tensor([3]))
