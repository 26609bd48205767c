"""CPU: the product's host-side logic (schedule tables, respacing, drop-in API surface, C-ABI symbol table)."""
import argparse
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, golden
from rohm_b200 import _lib, diffusion, schedule, synthetic

TABLES = schedule.TABLE_NAMES


def _make(sched, steps, resp, cls=diffusion.SpacedDiffusionPoseNet):
    args = argparse.Namespace(noise_schedule=sched, sigma_small=True)
    return diffusion.create_gaussian_diffusion(args, diffusion, cls, steps, resp, 'cpu')


def test_tables_and_timestep_maps_bit_exact_vs_reference():
    g = golden("schedules.npz")
    for c in range(int(g["n_cases"])):
        sched, steps, resp = [str(x) for x in g[f"c{c}_meta"]]
        for cls in (diffusion.SpacedDiffusionPoseNet, diffusion.SpacedDiffusionTrajNet):
            d = _make(sched, int(steps), resp, cls)
            assert d.timestep_map == g[f"c{c}_timestep_map"].tolist()
            assert d.num_timesteps == len(d.timestep_map)
            for t in TABLES:
                assert np.array_equal(getattr(d, t), g[f"c{c}_{t}"]), (sched, steps, resp, t)


def test_space_timesteps_bit_exact_and_errors():
    g = golden("schedules.npz")
    assert sorted(schedule.space_timesteps(300, [10, 15, 20])) == g["space_300_10_15_20"].tolist()
    assert sorted(schedule.space_timesteps(1000, "ddim100")) == g["space_1000_ddim100"].tolist()
    assert sorted(schedule.space_timesteps(1000, "100")) == g["space_1000_100"].tolist()
    assert sorted(schedule.space_timesteps(1000, "7,13,29")) == g["space_1000_7_13_29"].tolist()
    with pytest.raises(ValueError):
        schedule.space_timesteps(1000, "ddim300")
    with pytest.raises(ValueError):
        schedule.space_timesteps(10, [20])
    assert schedule.space_timesteps(5, [1]) == {0}
    with pytest.raises(NotImplementedError):
        schedule.get_named_beta_schedule("sqrt", 10)


def test_coef_rows_are_the_fp32_rounded_tables():
    d = _make("cosine", 1000, "")
    rows = schedule.ddpm_coef_rows({t: getattr(d, t) for t in TABLES})
    assert rows.dtype == np.float32 and rows.shape == (1000, 8)
    assert rows[0, 0] == 1.0 and rows[0, 1] == 0.0 and rows[0, 2] == 0.0  # final step: x_{-1} = x0 exactly, no noise
    assert np.array_equal(rows[:, 0], d.posterior_mean_coef1.astype(np.float32))
    assert np.array_equal(rows[:, 3], d.posterior_variance.astype(np.float32))
    lv = torch.from_numpy(d.posterior_log_variance_clipped).float()
    assert np.allclose(rows[1:, 2], torch.exp(0.5 * lv)[1:].numpy(), rtol=2e-7, atol=0)
    # Appendix F fp32-extracted coef1[[0,50,999]]
    assert [float(rows[i, 0]) for i in (0, 50, 999)] == [1.0, 0.03428633511066437, 0.0015568917151540518]


def test_wrapped_model_maps_timesteps_bit_exact():
    d = _make("cosine", 1000, "ddim100")
    seen = {}

    class M:
        def __call__(self, batch, ts):
            seen["ts"] = ts.clone()
            return batch

    w = d._wrap_model(M())
    ts = torch.tensor([0, 5, 99, 42])
    w({}, ts)
    assert seen["ts"].dtype == torch.int64 and seen["ts"].tolist() == [0, 50, 990, 420]
    assert d._wrap_model(w) is w
    assert d._scale_timesteps(ts) is ts


def test_dropin_packages_shadow_reference_names():
    dropin = os.path.join(ROOT, "rohm_b200", "dropin")
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r);"
            "import diffusion.gaussian_diffusion_posenet as gp, diffusion.gaussian_diffusion_trajnet as gt;"
            "import diffusion.respace as rs, utils.model_util as mu, model.posenet as mp, model.trajnet as mt;"
            "import model.cfg_sampler as cs, model.heads as mh;"
            "assert hasattr(gp, 'get_named_beta_schedule') and hasattr(gp, 'GaussianDiffusionPoseNet');"
            "assert hasattr(gt, 'GaussianDiffusionTrajNet') and hasattr(gp, 'LossType') and hasattr(gp, 'ModelMeanType');"
            "assert hasattr(rs, 'SpacedDiffusionPoseNet') and hasattr(rs, 'SpacedDiffusionTrajNet') and hasattr(rs, 'space_timesteps');"
            "assert hasattr(mu, 'create_gaussian_diffusion') and hasattr(mp, 'PoseNet') and hasattr(mt, 'TrajNet');"
            "assert hasattr(cs, 'ClassifierFreeSampleModel') and hasattr(mh, 'ResidualTemporalBlock');"
            "import rohm_b200; assert 'rohm_b200' in gp.__file__ or 'dropin' in gp.__file__; print('ok')") % (ROOT, dropin)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stderr[-2000:]


def test_posenet_and_trajnet_state_dict_keys_and_param_counts():
    from rohm_b200.posenet import PoseNet
    from rohm_b200.trajnet import TrajNet
    ds = synthetic.make_dataset('pose')
    m = PoseNet(dataset=ds, body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4, device=None,
                traj_feat_dim=22)
    n = sum(p.numel() for k, p in m.named_parameters() if not k.startswith("smplx_model."))
    assert n == 17789200  # SURVEY.md Appendix F
    keys = set(m.state_dict().keys())
    for k in ("input_process.poseEmbedding.weight", "input_process_cond.poseEmbedding.bias", "sequence_pos_encoder.pe",
              "embed_timestep.sequence_pos_encoder.pe", "embed_timestep.time_embed.2.weight",
              "seqTransEncoder.layers.7.self_attn.in_proj_weight", "seqTransEncoder.layers.0.norm2.bias",
              "output_process.poseFinal.weight"):
        assert k in keys, k
    dt = synthetic.make_dataset('traj')
    t0 = TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=False, dataset=dt, repr_abs_only=True)
    t1 = TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=True, dataset=dt, repr_abs_only=True)
    assert sum(p.numel() for p in t0.parameters()) == 22582893
    assert sum(p.numel() for p in t1.parameters()) == 37825450
    k1 = set(t1.state_dict().keys())
    for k in ("controlnet.control_zero_conv_0.weight", "controlnet.control_enc1.blocks.0.block.2.weight",
              "controlnet.control_mid_block1.residual_conv.bias", "time_mlp.3.weight", "diff_enc1.time_mlp.1.weight",
              "diff_upsample4.conv.weight", "diff_final_conv.1.bias", "cond_downsample4.conv.weight",
              "diff_final_conv.0.block.0.weight"):
        assert k in k1, k
    assert float(t1.controlnet.control_zero_conv_mid.weight.abs().max()) == 0.0  # zero-initialised


def test_no_cpu_fallback():
    from rohm_b200.posenet import PoseNet
    ds = synthetic.make_dataset('pose')
    m = PoseNet(dataset=ds, body_feat_dim=294, latent_dim=512, device=None, traj_feat_dim=22).eval()
    with pytest.raises(_lib.RohmB200Error):
        m({'x_t': torch.zeros(1, 294, 1, 8), 'cond': torch.zeros(1, 294, 1, 8)}, torch.zeros(1, dtype=torch.long))
    d = _make("cosine", 10, "")
    with pytest.raises(_lib.RohmB200Error):
        d.p_sample(lambda b, t: b['x_t'], {}, torch.zeros(1, 4), torch.zeros(1, dtype=torch.long))


def test_c_abi_library_exports_every_declared_symbol():
    """include/rohm_b200.h <-> librohm_b200.so <-> the ctypes signature table (no compute calls here): the same names, and
    each declaration's parameter count equal to its argtypes count (a list one pointer short would pass every argument
    after it in the wrong place)."""
    header = open(os.path.join(ROOT, "include", "rohm_b200.h")).read()
    params = dict(re.findall(r"ROHM_API\s+[\w\s\*]+?\b(rohm_\w+)\s*\(([^)]*)\)", header))
    declared = set(params)
    assert declared, "no declarations parsed"
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    for name, plist in params.items():
        plist = " ".join(plist.split())
        count = 0 if plist in ("", "void") else plist.count(",") + 1
        assert count == len(_lib.SIGNATURES[name][1]), (name, count, len(_lib.SIGNATURES[name][1]))
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.rohm_version() >= 101


def test_precision_modes_env_and_header_agree(monkeypatch):
    """ROHM_B200_PRECISION parsing and the enum values shared between include/rohm_b200.h and the ctypes layer."""
    from rohm_b200.posenet import _precision_from_env
    header = open(os.path.join(ROOT, "include", "rohm_b200.h")).read()
    for name, const in (("ROHM_PRECISION_TF32X3", _lib.PRECISION_TF32X3), ("ROHM_PRECISION_F16X2", _lib.PRECISION_F16X2),
                        ("ROHM_PRECISION_TF32", _lib.PRECISION_TF32)):
        m = re.search(name + r"\s*=\s*(\d+)", header)
        assert m and int(m.group(1)) == const, name
    monkeypatch.delenv("ROHM_B200_PRECISION", raising=False)
    assert _precision_from_env() == _lib.PRECISION_F16X2                      # default: fp16 hi/lo pairs
    assert _precision_from_env(supports_f16=False) == _lib.PRECISION_TF32X3  # engines without an fp16 path
    for text, want in (("tf32x3", _lib.PRECISION_TF32X3), ("F16X2", _lib.PRECISION_F16X2), ("tf32", _lib.PRECISION_TF32),
                       ("fast", _lib.PRECISION_TF32)):
        monkeypatch.setenv("ROHM_B200_PRECISION", text)
        assert _precision_from_env() == want
    monkeypatch.setenv("ROHM_B200_PRECISION", "bf16")
    with pytest.raises(_lib.RohmB200Error):
        _precision_from_env()


def test_body_model_create_refuses_a_missing_model_file(tmp_path):
    """A non-empty body_model_path without smplx/SMPLX_NEUTRAL.npz must raise (round-1 finding: it silently built the
    synthetic body); the synthetic model is an explicit opt-in."""
    from rohm_b200._lib import RohmB200Error
    from rohm_b200.body_model import BodyModel
    with pytest.raises(RohmB200Error):
        BodyModel.create(str(tmp_path / "no_such_dir"))
    assert BodyModel.create('').v_template.shape == (10475, 3)
    assert BodyModel.create(str(tmp_path), synthetic_ok=True).posedirs.shape == (486, 10475 * 3)
    # official layout: <path>/smplx/SMPLX_NEUTRAL.npz
    m = synthetic.smplx_like_model(1, num_verts=64)
    os.makedirs(tmp_path / "smplx")
    sd = np.zeros((64, 3, 400), np.float32)
    sd[:, :, :10], sd[:, :, 300:310] = m["shapedirs"][:, :, :10].numpy(), m["shapedirs"][:, :, 10:].numpy()
    kt = np.stack([np.array([2 ** 32 - 1] + m["parents"][1:], dtype=np.int64), np.arange(55)])
    np.savez(tmp_path / "smplx" / "SMPLX_NEUTRAL.npz", v_template=m["v_template"].numpy(), shapedirs=sd,
             posedirs=m["posedirs"].numpy().T.reshape(64, 3, 486), J_regressor=m["J_regressor"].numpy(),
             weights=m["lbs_weights"].numpy(), kintree_table=kt)
    b = BodyModel.create(str(tmp_path))
    assert torch.equal(b.posedirs, m["posedirs"]) and torch.equal(b.shapedirs, m["shapedirs"])
    assert b.parents.tolist() == m["parents"]


def test_posenet_adopts_smplx_buffers_of_a_reference_checkpoint():
    """A reference checkpoint stores the whole smplx module under smplx_model.* (more buffers than RoHM's calls read);
    strict loading must succeed and the body tensors must be taken from the checkpoint."""
    from rohm_b200.posenet import PoseNet
    ds = synthetic.make_dataset('pose')
    m = PoseNet(dataset=ds, body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8, num_heads=4, device=None,
                traj_feat_dim=22)
    sd = synthetic.synth_state_dict(m, 1)
    body = synthetic.smplx_like_model(7)
    sd = {k: v for k, v in sd.items() if not k.startswith("smplx_model.")}
    sd.update({"smplx_model.v_template": body["v_template"], "smplx_model.shapedirs": body["shapedirs"][:, :, :10],
               "smplx_model.expr_dirs": body["shapedirs"][:, :, 10:], "smplx_model.posedirs": body["posedirs"],
               "smplx_model.J_regressor": body["J_regressor"], "smplx_model.lbs_weights": body["lbs_weights"],
               "smplx_model.parents": torch.tensor([-1] + body["parents"][1:]),
               "smplx_model.faces_tensor": torch.zeros(20908, 3, dtype=torch.long),
               "smplx_model.global_orient": torch.zeros(1, 3), "smplx_model.pose_mean": torch.zeros(165)})
    res = m.load_state_dict(sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    assert torch.equal(m.smplx_model.v_template, body["v_template"])
    assert torch.equal(m.smplx_model.shapedirs, body["shapedirs"])
    # own-format state dicts still round-trip
    m.load_state_dict(m.state_dict(), strict=True)


def test_sampler_guards_fire_before_any_denoiser_call():
    """DDIM respacing with guidance / early-stop and a timestep map beyond the positional table are rejected up front."""
    from rohm_b200._lib import RohmB200Error

    class Boom:
        def parameters(self):
            raise AssertionError("the sampler touched the model before validating its arguments")

        def __call__(self, *a, **k):
            raise AssertionError("denoiser called")

    d = _make('cosine', 1000, 'ddim10')
    for kw in (dict(cond_fn_with_grad=True, grad_type='amass'), dict(early_stop=True)):
        with pytest.raises(RohmB200Error):
            d.eval_losses(model=Boom(), batch={}, shape=[1, 294, 1, 8], timestep_respacing='ddim10', compute_loss=False, **kw)


def test_dropin_motion_representation_keeps_the_reference_symbols(tmp_path):
    """dropin/data_loaders/motion_representation.py shadows only recover_from_repr_smpl; every other symbol of the
    reference's module (found further down sys.path) is re-exported, and data_loaders.common still resolves to the reference
    tree (namespace-package merge).  A stand-in 'reference' tree is used: the real one is not on the GPU box."""
    ref = tmp_path / "ref"
    (ref / "data_loaders" / "common").mkdir(parents=True)
    (ref / "data_loaders" / "common" / "__init__.py").write_text("")
    (ref / "data_loaders" / "common" / "quaternion.py").write_text("def qinv(q):\n    return 'ref-qinv'\n")
    (ref / "data_loaders" / "motion_representation.py").write_text(
        "from data_loaders.common.quaternion import *\n"
        "def get_repr_smplx(*a, **k):\n    return 'ref-get_repr'\n"
        "def recover_from_repr_smpl(data_dict, recover_mode='joint_abs_traj', smplx_model=None, return_verts=False,"
        " return_full_joints=False):\n    return 'ref-recover'\n")
    dropin = os.path.join(ROOT, "rohm_b200", "dropin")
    code = ("import sys; sys.path[:0] = [%r, %r, %r];"
            "import torch;"
            "from data_loaders.motion_representation import *;"
            "import data_loaders.motion_representation as mr, data_loaders.common.quaternion as q;"
            "assert 'dropin' in mr.__file__ and get_repr_smplx() == 'ref-get_repr' and qinv(0) == 'ref-qinv';"
            "assert recover_from_repr_smpl({'a': torch.zeros(1, 2, 1)}) == 'ref-recover';"  # CPU tensors: the reference's own code
            "print('ok')") % (dropin, ROOT, str(ref))
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stderr[-2000:]
