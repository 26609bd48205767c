"""Host-side checks of the per-clip guidance normalisers (PoseNet.guidance_normaliser = 'clip'); no GPU: the C ABI of the two
guidance entry points, the float64 per-clip oracles against the reference's one-clip runs (tests/golden/clip_guidance.npz,
tools/gen_golden.py clip_guidance), and the refusals."""
import argparse
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from helpers import ROOT, golden
from oracle import clip_guidance_oracle as cgo
from rohm_b200 import _lib, diffusion, parallel, synthetic
from rohm_b200._lib import RohmB200Error
from rohm_b200.posenet import PoseNet


def _declaration(header, name):
    m = re.search(r"ROHM_API\s+[\w\s\*]+?\b" + name + r"\s*\(([^)]*)\)", header)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


def test_guidance_entry_points_take_the_per_clip_switch():
    header = open(os.path.join(ROOT, "include", "rohm_b200.h")).read()
    sk = _declaration(header, "rohm_skating_guidance")
    pj = _declaration(header, "rohm_projection_guidance")
    assert "int per_clip" in sk and "const int* lengths" in sk
    assert "int per_clip" in pj and "const int* lengths" in pj
    # lengths and per_clip sit where the ctypes table has a pointer and an int
    for params, name in ((sk, "rohm_skating_guidance"), (pj, "rohm_projection_guidance")):
        argtypes = _lib.SIGNATURES[name][1]
        assert len(params) == len(argtypes), name
        assert argtypes[params.index("const int* lengths")] is ctypes.c_void_p, name
        assert argtypes[params.index("int per_clip")] is ctypes.c_int, name
    # the two halves for batch-global normalisers are unchanged
    assert "int per_clip" not in _declaration(header, "rohm_skating_guidance_sums")
    assert "int per_clip" not in _declaration(header, "rohm_skating_guidance_backward")
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    assert hasattr(lib, "rohm_skating_guidance") and hasattr(lib, "rohm_projection_guidance")
    assert lib.rohm_version() >= 102


def _fixture():
    g = golden("clip_guidance.npz")
    ds = synthetic.make_dataset('pose', seed=int(g["ds_seed"]), realistic_std=True)
    t = lambda k: torch.from_numpy(g[k])
    return g, ds, t


def test_per_clip_skating_oracle_matches_the_reference_on_each_clip_alone():
    g, ds, t = _fixture()
    lengths = [int(v) for v in g["lengths"]]
    grad = cgo.guide_skating_per_clip(t("x"), torch.from_numpy(ds.Mean), torch.from_numpy(ds.Std),
                                      synthetic.smplx_like_model(0), lengths)
    ref = g["skating_grad"]
    assert np.isfinite(grad.numpy()).all(), "a padded NaN reached the gradient"
    assert np.abs(grad.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())
    for b, n in enumerate(lengths):
        skates = bool(g["skates"][b])
        assert (np.abs(ref[b, ..., :n]).max() > 0) == skates, b
        assert not grad[b, ..., n:].any(), b
    assert list(g["skates"]) == [1, 1, 0, 0], "the fixture has two skating clips and two without a skating frame"


def test_per_clip_projection_oracle_matches_the_reference_on_each_clip_alone():
    g, ds, t = _fixture()
    lengths = [int(v) for v in g["lengths"]]
    grad, loss = cgo.guide_projection_per_clip(t("x"), torch.from_numpy(ds.Mean), torch.from_numpy(ds.Std),
                                               synthetic.smplx_like_model(0), t("transf"), t("cam_R"), t("cam_t"),
                                               t("focal"), t("center"), t("kp"), lengths)
    ref = g["proj_grad"]
    assert loss.shape == (len(lengths),) and bool(torch.isfinite(loss).all())
    assert np.abs(grad.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())
    assert np.abs(ref[:, 0:22]).max() == 0 and np.abs(ref[:, -4:]).max() == 0
    for b, n in enumerate(lengths):
        assert np.abs(ref[b, ..., :n]).max() > 0, b
        assert not grad[b, ..., n:].any(), b


def _model():
    ds = synthetic.make_dataset('pose')
    return PoseNet(dataset=ds, body_feat_dim=294, latent_dim=512, device=None, traj_feat_dim=22).eval()


def _diffusion():
    args = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    return diffusion.create_gaussian_diffusion(args, diffusion, diffusion.SpacedDiffusionPoseNet, 1000, '10', 'cpu')


def test_the_mode_is_a_plain_attribute():
    m = _model()
    assert m.guidance_normaliser == 'batch' and not m.guidance_per_clip()
    m.guidance_normaliser = 'clip'
    assert m.guidance_per_clip()
    assert not any("guidance_normaliser" in k for k in m.state_dict())
    m.load_state_dict(m.state_dict())
    m = m.to(torch.float32)
    assert m.guidance_normaliser == 'clip'


@pytest.mark.parametrize("bad", ['Clip', 'per_clip', None, 1, ''])
def test_a_bad_mode_is_refused_before_anything_runs(bad):
    m = _model()
    m.guidance_normaliser = bad
    d = _diffusion()
    x = torch.zeros(2, 294, 1, 8)
    with pytest.raises(RohmB200Error, match="guidance_normaliser"):
        d.p_sample_loop(m, {'cond': x}, [2, 294, 1, 8], cond_fn_with_grad=True, grad_type='amass')
    for hook in (m.guide_skating_with_smpl, m.guide_2d_projection_with_smpl):
        with pytest.raises(RohmB200Error, match="guidance_normaliser"):
            hook({'x_t': x}, {'pred_xstart': x}, None, compute_grad='x_0')


def test_clip_mode_and_global_guidance_are_refused_in_either_order():
    m = _model()
    m.guidance_normaliser = 'clip'
    with pytest.raises(RohmB200Error, match="guidance_normaliser='clip'"):
        parallel.global_guidance(m)
    assert not hasattr(m, "guidance_sum_reducer")
    parallel.global_guidance(m, enable=False)  # disabling is always allowed

    m = _model()
    parallel.global_guidance(m)
    m.guidance_normaliser = 'clip'
    x = torch.zeros(2, 294, 1, 8)
    with pytest.raises(RohmB200Error, match="global_guidance"):
        _diffusion().p_sample_loop(m, {'cond': x}, [2, 294, 1, 8], cond_fn_with_grad=True, grad_type='prox')
    with pytest.raises(RohmB200Error, match="global_guidance"):
        m.guide_skating_with_smpl({'x_t': x}, {'pred_xstart': x}, None, compute_grad='x_0')
    parallel.global_guidance(m, enable=False)
    assert m.guidance_per_clip()


def test_prox_with_lengths_is_accepted_in_clip_mode_only():
    m = _model()
    batch = {'lengths': torch.tensor([8, 5])}
    shape = (2, 294, 1, 8)
    with pytest.raises(RohmB200Error, match="prox"):
        m.clip_lengths(batch, shape, grad_type='prox')
    m.guidance_normaliser = 'clip'
    assert m.clip_lengths(batch, shape, grad_type='prox') == (8, 5)
    assert m.clip_lengths(batch, shape, grad_type='amass') == (8, 5)
