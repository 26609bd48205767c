"""CPU: pins the video driver's oracle (oracle/video_pipeline_oracle.py) to the golden produced by the unmodified reference
(tools/gen_golden.py:gen_video_pipeline -> tests/golden/video_pipeline.npz): one PROX and one EgoBody recording, each cut
into two short windows by the reference's own video loader, through 2 rounds of the PROX / EgoBody driver."""
import numpy as np
import pytest
import torch

from helpers import NoiseTape, TOL, golden
from oracle import video_pipeline_oracle
from rohm_b200 import synthetic
from rohm_b200.windows import ABS_TRAJ_CHANNELS

POSE_RESPACING = "12" + ",0" * 19  # tools/gen_golden.py POSE_RESPACING: 12 guided steps inside t < 50
NOISE_SEEDS = lambda c: (130 + c, 140 + c)  # gen_video_pipeline's PoseNet / TrajNet noise tapes


def case_inputs(g, c):
    """(pose batch, traj batch, camera) of case c as CPU tensors: the loader's keys the driver reads."""
    t = lambda k: torch.from_numpy(g[k])
    pose = {k[len(f"c{c}_pose_"):]: t(k) for k in g.files if k.startswith(f"c{c}_pose_")}
    traj = {'motion_repr_noisy': t(f"c{c}_traj_motion_repr_noisy")}
    traj['cond'] = traj['motion_repr_noisy'][..., list(ABS_TRAJ_CHANNELS)]  # the loader's repr_abs_only channels
    traj['control_cond'] = traj['motion_repr_noisy'][..., -272:].contiguous()
    c2w = t(f"c{c}_cam2world")
    camera = {'transf_matrix': pose['transf_matrix'], 'cam_R': c2w[:3, :3], 'cam_t': c2w[:3, 3].reshape(1, 3),
              'focal_length': pose['focal_length'], 'camera_center': pose['camera_center'],
              'keypoints_2d': pose['keypoints_2d']}
    return pose, traj, camera


def teacher(g, c):
    return {k[len(f"c{c}_"):]: g[k] for k in g.files if k.startswith(f"c{c}_r")}


@pytest.mark.parametrize("case", [0, 1])
def test_video_oracle_matches_reference_rounds(case):
    from rohm_b200.posenet import PoseNet
    from rohm_b200.trajnet import TrajNet
    g = golden("video_pipeline.npz")
    _, tn, pn, rounds, _, _ = [int(v) for v in g["meta"]]
    steps = tuple(int(v) for v in g["recorded_steps"])
    ds_pose = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_traj = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    sd_pose = synthetic.synth_state_dict(PoseNet(dataset=ds_pose, body_feat_dim=294, latent_dim=512, traj_feat_dim=22), 1)
    mk = lambda c: TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=c, repr_abs_only=True)
    sd_traj, sd_ctrl = synthetic.synth_state_dict(mk(False), 2), synthetic.synth_state_dict(mk(True), 4)
    pose, traj, camera = case_inputs(g, case)
    s_pose, s_traj = NOISE_SEEDS(case)
    res = video_pipeline_oracle.run_video_rounds(sd_pose, sd_traj, sd_ctrl, ds_pose, ds_traj, synthetic.smplx_like_model(0),
                                                 pose, traj, 1000, tn, rounds, NoiseTape(s_pose), NoiseTape(s_traj), camera,
                                                 pose_respacing=POSE_RESPACING, teacher=teacher(g, case),
                                                 teacher_steps=steps)
    assert pn == 12 and steps == (1, 0)
    for it in range(rounds):
        ref = lambda k: g[f"c{case}_r{it}_{k}"]
        err = {k: float(np.abs(res[it][k].numpy() - ref(k)).max()) for k in ("val_traj", "traj_full", "cond", "val_pose")}
        tf = res[it]['tf']
        # teacher-forced: x_1 -> x_0 (guided, relative bound) and x_0 -> the early-stopped output pred_xstart (absolute)
        e10 = float((tf[1] - torch.from_numpy(ref("xt0"))).abs().max()) / float(np.abs(ref("xt0")).max())
        e0 = float((tf[0] - torch.from_numpy(ref("val_pose"))).abs().max())
        print(f"case {case} round {it}: stages {err} | teacher-forced: step1 rel {e10:.2e}, final abs {e0:.2e}")
        assert err["val_traj"] < TOL and err["traj_full"] < TOL and err["cond"] < TOL, (it, err)
        assert e10 < 1e-3 and e0 < TOL, (it, e10, e0)
