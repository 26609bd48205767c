"""GPU: the PROX / EgoBody video driver's rounds on the device (pipeline.run_video_rounds, reconstruct_video_outputs,
video_result_dicts and the visibility-masked PoseNet condition of glue.build_pose_cond), replayed against the golden the
unmodified reference produced on windows of its own video loader (tests/golden/video_pipeline.npz,
tools/gen_golden.py:gen_video_pipeline), and run on windows of several recordings at once."""
import numpy as np
import pytest
import torch

import test_gpu_pipeline as tp
from helpers import NoiseTape, TOL, golden
from rohm_b200 import glue, pipeline, synthetic, windows
from rohm_b200._lib import RohmB200Error
from rohm_b200.body_model import BodyModel
from test_gpu_noise_streams import _clone, _gens
from test_gpu_windows import _recording_params
from test_oracle_video_pipeline_golden import NOISE_SEEDS, case_inputs

pytestmark = pytest.mark.gpu

VIDEO_ARGS = dict(sample_iter=2, iter2_cond_noisy_traj=False, iter2_cond_noisy_pose=False, early_stop=True)
REC_KEYS = ('rec_ric_data_noisy', 'rec_ric_data_rec_from_abs_traj', 'rec_ric_data_rec_from_smpl', 'smpl_verts_rec',
            'smpl_verts_noisy', 'motion_repr_rec', 'motion_repr_noisy')


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.fixture(scope="module")
def nets(cuda_device):
    ds_p = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    ds_t = synthetic.make_dataset('traj', seed=3, realistic_std=True)
    mp, mt, mc, *_ = tp._models(cuda_device, ds_p, ds_t)
    return ds_p, ds_t, mp, mt, mc, BodyModel.create('', device=cuda_device, seed=0)


# ---------------------------------------------------------------------------------------------- 1. reference replay
def _fixture_batches(g, c, dev):
    pose, traj, camera = case_inputs(g, c)
    pose = {k: v.to(dev) for k, v in pose.items()}
    traj = {k: v.to(dev) for k, v in traj.items()}
    pose['cam2world'] = torch.from_numpy(g[f"c{c}_cam2world"]).to(dev).repeat(pose['transf_matrix'].shape[0], 1, 1)
    return pose, traj


@pytest.mark.parametrize("case", [0, 1])
def test_video_rounds_replay_reference_golden(nets, cuda_device, case):
    dev = cuda_device
    ds_p, ds_t, mp, mt, mc, body = nets
    g = golden("video_pipeline.npz")
    _, tn, pn, rounds, _, _ = [int(v) for v in g["meta"]]
    s_pose, s_traj = NOISE_SEEDS(case)
    dp, dt, dc = tp._diffusions(dev, tn)
    tape_p, tape_t = NoiseTape(s_pose, dev), NoiseTape(s_traj, dev)
    dp._randn, dp._randn_like = tape_p.randn, tape_p.randn_like
    for d in (dt, dc):  # the reference's two TrajNet diffusion objects share one module-level RNG stream
        d._randn, d._randn_like = tape_t.randn, tape_t.randn_like
    pose, traj = _fixture_batches(g, case, dev)
    B, T = traj['motion_repr_noisy'].shape[0], traj['motion_repr_noisy'].shape[1]  # the fixture's short windows
    ref = lambda it, k: torch.from_numpy(g[f"c{case}_r{it}_{k}"])
    seen = []

    def on_round(it, val_traj, traj_full, cond, val_pose):
        seen.append({k: v.detach().cpu() for k, v in (("val_traj", val_traj), ("traj_full", traj_full), ("cond", cond),
                                                      ("val_pose", val_pose))})
        return ref(it, "val_pose").to(dev)  # stage-wise: the next round starts from the reference's PoseNet output

    out_pose, out_traj = pipeline.run_video_rounds(pipeline.make_args(**VIDEO_ARGS), mp, mt, mc, dp, dt, dc, ds_p, ds_t, body,
                                                   pose, traj, on_round=on_round)
    assert out_pose.shape == (B, 294, 1, T - 1) and out_traj.shape == (B, T, 13)
    fresh_pose, fresh_traj = _fixture_batches(g, case, dev)
    base = fresh_traj['motion_repr_noisy']
    for it in range(rounds):
        # TrajNet free-running (round 1 on the reference's round-0 PoseNet output)
        e_traj = float((seen[it]['val_traj'] - ref(it, "val_traj")).abs().max())
        # the glue on the reference's TrajNet output; round 1 builds on round 0's composite
        comp, tf_full = glue.traj_to_full_repr(body, ref(it, "val_traj").to(dev), base, ds_t, ds_p)
        if it == 0:
            base = comp
        e_full = float((tf_full.cpu() - ref(it, "traj_full")).abs().max())
        # the condition on the reference's trajectory block and source: bit-equal
        if it == 0:
            cond = glue.build_pose_cond(fresh_pose['motion_repr_noisy'][:, 0:-1], ref(it, "traj_full").to(dev),
                                        zero_contact=True, vis_mask=fresh_pose['mask_vec_vis'])
        else:
            cond = glue.build_pose_cond(ref(it - 1, "val_pose").to(dev), ref(it, "traj_full").to(dev))
        print(f"case {case} round {it}: val_traj {e_traj:.2e}, traj_full (stage-wise) {e_full:.2e}")
        assert e_traj < TOL and e_full < TOL, (it, e_traj, e_full)
        assert torch.equal(_bits(cond.cpu()), _bits(ref(it, "cond"))), it
    # teacher-forced guided PoseNet steps from the reference's recorded states (grad_type 'prox', every step guided)
    t_rows = dp._t_rows(B, dev)
    for it in range(rounds):
        tape = NoiseTape(s_pose, dev)
        for _ in range(it * (pn + 1) + 1):
            tape.randn(B, 294, 1, T - 1)  # earlier rounds' draws and this round's x_T
        noises = {i: tape.randn(B, 294, 1, T - 1) for i in range(pn - 1, -1, -1)}
        batch = {k: pose[k] for k in ('transf_matrix', 'focal_length', 'camera_center', 'keypoints_2d', 'cam2world')}
        batch['cond'] = ref(it, "cond").to(dev)
        for i, nxt in ((1, "xt0"), (0, "val_pose")):
            dp._randn_like = lambda x, _n=noises[i]: _n
            o = dp.p_sample_with_grad(mp, batch, ref(it, f"xt{i}").to(dev), t_rows[i], clip_denoised=False, grad_type='prox',
                                      _step_index=i)
            got = o['pred_xstart'] if i == 0 else o['sample']  # early_stop returns the last step's pred_xstart
            err = float((got.cpu() - ref(it, nxt)).abs().max())
            rel = err / float(ref(it, nxt).abs().max())
            print(f"case {case} round {it} guided step i={i}: teacher-forced max err {err:.3e} (rel {rel:.2e})")
            assert (err < TOL) if i == 0 else (rel < 1e-3), (it, i, err, rel)
    # the reconstruction of the reference's final output
    noisy = fresh_pose['motion_repr_noisy'][:, 0:-1].permute(0, 2, 1).unsqueeze(-2)
    rec = pipeline.reconstruct_video_outputs(ds_p, body, {'motion_repr_noisy': noisy}, ref(rounds - 1, "val_pose").to(dev))
    for key, gk in (('rec_ric_data_noisy', 'rec_noisy'), ('rec_ric_data_rec_from_abs_traj', 'rec_from_abs_traj'),
                    ('rec_ric_data_rec_from_smpl', 'rec_from_smpl')):
        err = float((rec[key].cpu() - torch.from_numpy(g[f"c{case}_{gk}"])).abs().max())
        print(f"case {case} reconstruction {key}: {err:.2e}")
        assert err < TOL, (key, err)


# ---------------------------------------------------------------------------------------------- 2. condition bits
def _specials(shape, seed, dev):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=gen)
    pick = torch.randint(0, 8, shape, generator=gen)
    x[pick == 0] = -0.0
    x[pick == 1] = float("nan")
    x[pick == 2] = float("inf")
    x[pick == 3] = -float("inf")
    x[pick == 4] = -x[pick == 4].abs()  # negative finite: x * 0 = -0.0
    return x.to(dev)


def test_condition_kernel_matches_the_torch_expression(cuda_device):
    """test_prox_egobody.py:302-309 as torch evaluates it on the device, bit for bit (NaN payloads included)."""
    dev = cuda_device
    B, Tp = 3, 143
    src_cl = _specials((B, Tp + 1, 294), 1, dev)
    traj_full = _specials((B, Tp, 22), 2, dev)
    gen = torch.Generator().manual_seed(3)
    vis = (torch.rand(B, 145, 294, generator=gen) > 0.3).float()
    vis[0, 5, 40] = 0.5
    vis = vis.to(dev)
    for zero_contact in (True, False):
        want = src_cl[:, 0:Tp].clone()
        want[:, :, 0:22] = traj_full
        want = want * vis[:, 0:-2, :]
        if zero_contact:
            want[:, :, -4:] = 0.
        want = torch.permute(want, (0, 2, 1)).unsqueeze(-2)
        got_cl = glue.build_pose_cond(src_cl, traj_full, zero_contact=zero_contact, frames=Tp, vis_mask=vis)
        src_cm = src_cl[:, 0:Tp].permute(0, 2, 1).unsqueeze(-2).contiguous()
        got_cm = glue.build_pose_cond(src_cm, traj_full, zero_contact=zero_contact, vis_mask=vis)
        assert torch.equal(_bits(got_cl), _bits(want)), zero_contact
        assert torch.equal(_bits(got_cm), _bits(want)), zero_contact
    assert bool(torch.isnan(want).any()) and bool((_bits(want) == -2 ** 31).any())  # NaN and -0.0 did occur
    # without a mask the existing call is unchanged
    plain = glue.build_pose_cond(src_cl, traj_full, zero_contact=True, frames=Tp)
    assert not torch.equal(_bits(plain), _bits(got_cl))
    for bad in (vis[:, 0:Tp - 1], vis.double(), vis.cpu(), vis[0:2], vis[..., 0:293]):
        with pytest.raises(RohmB200Error):
            glue.build_pose_cond(src_cl, traj_full, frames=Tp, vis_mask=bad)
    with pytest.raises(RohmB200Error):
        glue.build_pose_cond(src_cl, traj_full, frames=Tp, vis_mask=vis,
                             lengths=torch.full((B,), Tp, dtype=torch.int32, device=dev))


# ---------------------------------------------------------------------------------------------- 3. many recordings
LENGTHS = (288, 145, 200)  # 2 + 1 + 1 windows of 145 frames


def _encode(dataset, nets, dev, with_gt=False):
    ds_p, ds_t, _, _, _, body = nets
    R, N = len(LENGTHS), sum(LENGTHS)
    recs = [_recording_params(n, 31 + i) for i, n in enumerate(LENGTHS)]
    params = {k: torch.from_numpy(np.concatenate([r[k] for r in recs])).to(dev) for k in recs[0]}
    params['transl'][:, 2] += 3.5  # camera-frame fits: every joint well in front of the camera, so projections are finite
    c2w = np.repeat(np.eye(4)[None], R, 0)
    for r in range(R):  # three different cameras
        a = 0.7 + r
        c2w[r, :3, :3] = [[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]]
        c2w[r, :3, 3] = [0.3 * r, -1.2, 2.0 + 0.5 * r]
    gk = np.random.default_rng(5)
    kp = np.concatenate([gk.uniform(-200, 2100, (N, 25, 1)), gk.uniform(-100, 1200, (N, 25, 1)),
                         gk.uniform(0, 1, (N, 25, 1))], -1).astype(np.float32)
    depth = (gk.uniform(0, 1, (N, 25)) > 0.1).astype(np.float32)
    K = np.array([[1060.53, 0.0, 951.3], [0.0, 1060.38, 536.77], [0.0, 0.0, 1.0]])
    kw = dict(cam2world=c2w, focal_length=np.repeat([[1060.53, 1060.38]], R, 0) + np.arange(R)[:, None],
              camera_center=np.repeat([[951.3, 536.77]], R, 0), camera_mtx=np.repeat(K[None], R, 0),
              dist=np.repeat([[0.0548, -0.0489, 0.0009, -0.0012, 0.0102]], R, 0), keypoints=torch.from_numpy(kp).to(dev),
              depth_mask=torch.from_numpy(depth).to(dev))
    if with_gt:
        kw.update(gt_params=params, gt_body_model=body, master2world=c2w)
    return windows.encode_video(body, params, LENGTHS, dataset, pose_dataset=ds_p, traj_dataset=ds_t, **kw)


def _take(batch, idx):
    return {k: ({a: b[idx] for a, b in v.items()} if isinstance(v, dict) else v[idx]) for k, v in batch.items()}


def _run(nets, dev, traj, pose, gens, args=None, invalidate=False):
    ds_p, ds_t, mp, mt, mc, body = nets
    dp, dt, dc = tp._diffusions(dev, 4, pose_steps=1000, pose_respacing="3" + ",0" * 19)
    if invalidate:
        mt.invalidate_engine()
        mc.invalidate_engine()
    traj = dict(traj, generators=gens)
    pose = dict(pose)
    conds = []
    vp, vt = pipeline.run_video_rounds(args or pipeline.make_args(**VIDEO_ARGS), mp, mt, mc, dp, dt, dc, ds_p, ds_t, body,
                                       pose, traj, on_round=lambda it, a, b, cond, d: conds.append(cond.clone()))
    rec = pipeline.reconstruct_video_outputs(ds_p, body, pose, vp)
    return vp, vt, conds, rec


@pytest.mark.parametrize("dataset", ['prox', 'egobody'])
def test_windows_of_many_recordings_run_as_if_alone(nets, cuda_device, dataset):
    dev = cuda_device
    mp, mt, mc = nets[2:5]
    bt, bp, win = _encode(dataset, nets, dev, with_gt=dataset == 'egobody')
    W = len(win)
    assert W == 4 and len(set(win.recording.tolist())) == 3
    seeds = [71 + w for w in range(W)]
    mp.guidance_normaliser, mt.batch_invariant, mc.batch_invariant = 'clip', True, True
    try:
        vp, vt, conds, rec = _run(nets, dev, bt, bp, _gens(dev, seeds))
        perm = [2, 0, 3, 1]
        pv, pt, pconds, prec = _run(nets, dev, _take(bt, perm), _take(bp, perm), _gens(dev, [seeds[p] for p in perm]))
        for w in range(W):
            ov, ot, oconds, orec = _run(nets, dev, _take(bt, [w]), _take(bp, [w]), _gens(dev, [seeds[w]]), invalidate=True)
            j = perm.index(w)
            for name, full, perm_, alone in (("val_pose", vp, pv, ov), ("val_traj", vt, pt, ot)):
                assert torch.equal(_bits(full[w:w + 1]), _bits(alone)), (w, name)
                assert torch.equal(_bits(perm_[j:j + 1]), _bits(alone)), (w, name, "permuted")
            for it in range(2):
                assert torch.equal(_bits(conds[it][w:w + 1]), _bits(oconds[it])), (w, it, "cond")
                assert torch.equal(_bits(pconds[it][j:j + 1]), _bits(oconds[it])), (w, it, "cond permuted")
            for key in REC_KEYS:
                assert torch.equal(_bits(rec[key][w:w + 1]), _bits(orec[key])), (w, key)
                assert torch.equal(_bits(prec[key][j:j + 1]), _bits(orec[key])), (w, key, "permuted")
    finally:
        mp.guidance_normaliser, mt.batch_invariant, mc.batch_invariant = 'batch', False, False
        mt.invalidate_engine()
        mc.invalidate_engine()
    assert all(bool(torch.isfinite(t).all()) for t in (vp, vt))


# ---------------------------------------------------------------------------------------------- 4. flags and payload
def test_flag_variants_and_batch_side_effects(nets, cuda_device):
    dev = cuda_device
    ds_p, ds_t, mp, mt, mc, body = nets
    bt, bp, win = _encode('prox', nets, dev)
    W = len(win)
    for noisy_pose, noisy_traj, early_stop in ((False, False, True), (True, False, True), (False, True, False),
                                               (True, True, False)):
        args = pipeline.make_args(sample_iter=2, iter2_cond_noisy_traj=noisy_traj, iter2_cond_noisy_pose=noisy_pose,
                                  early_stop=early_stop)
        traj, pose = dict(bt), dict(bp)
        noisy_rows, cond0 = traj['motion_repr_noisy'], traj['cond']
        dp, dt, dc = tp._diffusions(dev, 4, pose_steps=1000, pose_respacing="3" + ",0" * 19)
        seen, handed = [], []

        def on_round(it, *a):
            seen.append([t.clone() for t in a])
            handed.append(a[3])

        vp, vt = pipeline.run_video_rounds(args, mp, mt, mc, dp, dt, dc, ds_p, ds_t, body, pose, traj, on_round=on_round)
        assert vp.shape == (W, 294, 1, 143) and vt.shape == (W, 144, 13) and bool(torch.isfinite(vp).all())
        assert pose['motion_repr_noisy'].shape == (W, 294, 1, 143) and pose['cond'].shape == (W, 294, 1, 143)
        assert traj['control_cond'].shape == (W, 144, 272) and traj['motion_repr_noisy'].shape == (W, 144, 294)
        assert traj['motion_repr_noisy'] is not noisy_rows  # round 0's composite replaced the noisy rows
        if noisy_traj:
            assert traj['cond'] is cond0
        else:
            assert torch.equal(traj['cond'], seen[0][0])  # round 0's TrajNet output conditions round 1
        # round 1's condition: the noisy rows (masked, every round) or the previous output (unmasked)
        src = pose['motion_repr_noisy'] if noisy_pose else seen[0][3]
        want = glue.build_pose_cond(src, seen[1][1], zero_contact=noisy_pose,
                                    vis_mask=pose['mask_vec_vis'] if noisy_pose else None)
        assert torch.equal(_bits(seen[1][2]), _bits(want)), (noisy_pose, noisy_traj)
        assert torch.equal(_bits(handed[0]), _bits(seen[0][3]))  # an output handed to on_round is never written again


def test_result_dicts_split_per_recording(nets, cuda_device):
    dev = cuda_device
    ds_p, ds_t, mp, mt, mc, body = nets
    bt, bp, win = _encode('egobody', nets, dev, with_gt=True)
    W = len(win)
    dp, dt, dc = tp._diffusions(dev, 4, pose_steps=1000, pose_respacing="3" + ",0" * 19)
    vp, _ = pipeline.run_video_rounds(pipeline.make_args(**VIDEO_ARGS), mp, mt, mc, dp, dt, dc, ds_p, ds_t, body, bp, bt)
    rec = pipeline.reconstruct_video_outputs(ds_p, body, bp, vp)
    names = [[f"r{r}_frame_{i:05d}" for i in range(n)] for r, n in enumerate(LENGTHS)]
    payloads = pipeline.video_result_dicts(win, rec, bp, frame_names=names)
    world, covered = windows.to_recordings(win, rec['rec_ric_data_rec_from_smpl'])
    rec_ids, starts = win.recording.cpu().numpy(), win.start.cpu().numpy()
    assert len(payloads) == len(LENGTHS)
    total = 0
    for r, p in enumerate(payloads):
        idx = np.flatnonzero(rec_ids == r)
        n = len(idx)
        total += n
        order = idx[np.argsort(starts[idx])]
        shapes = {'trans_scene2cano_list': (n, 4, 4), 'rec_ric_data_noisy_list': (n, 143, 22, 3),
                  'rec_ric_data_rec_list_from_abs_traj': (n, 143, 22, 3), 'rec_ric_data_rec_list_from_smpl': (n, 143, 22, 3),
                  'joints_input_scene_coord_list': (n, 145, 22, 3), 'joints_gt_scene_coord_list': (n, 145, 22, 3),
                  'motion_repr_noisy_list': (n, 143, 294), 'motion_repr_rec_list': (n, 143, 294),
                  'mask_joint_vis_list': (n, 143, 22), 'frame_name_list': (n, 145)}
        assert set(p) == set(shapes) | {'repr_name_list', 'repr_dim_dict'}
        for k, s in shapes.items():
            assert p[k].shape == s, (r, k, p[k].shape)
        assert p['frame_name_list'][:, 0].tolist() == [names[r][s] for s in sorted(starts[idx])]
        assert np.array_equal(p['trans_scene2cano_list'], bp['transf_matrix'][torch.from_numpy(order)].cpu().numpy())
        wr, cr = world[r].cpu().double().numpy(), covered[r].cpu().numpy()
        for k, w in enumerate(order):
            inv = np.linalg.inv(p['trans_scene2cano_list'][k].astype(np.float64))
            j = p['rec_ric_data_rec_list_from_smpl'][k].astype(np.float64)
            scene = j @ inv[:3, :3].T + inv[:3, 3]
            s = int(starts[w])
            assert cr[s:s + 143].all()
            tol = 8 * np.finfo(np.float32).eps * (1 + np.abs(scene).max())
            assert np.abs(scene - wr[s:s + 143]).max() <= tol, (r, k)
    assert total == W
    assert 'frame_name_list' not in pipeline.video_result_dicts(win, rec, bp)[0]


class _Untouchable:
    def eval_losses(self, *a, **kw):
        raise AssertionError("a refused batch reached a sampling loop")


def test_refusals_before_any_sampling(nets, cuda_device):
    dev = cuda_device
    ds_p, ds_t, mp, mt, mc, body = nets
    bt, bp, win = _encode('prox', nets, dev)
    no = _Untouchable()
    run = lambda pose, traj: pipeline.run_video_rounds(pipeline.make_args(**VIDEO_ARGS), mp, mt, mc, no, no, no, ds_p, ds_t,
                                                       body, pose, traj)
    with pytest.raises(RohmB200Error, match="lengths"):
        run(dict(bp), dict(bt, lengths=torch.full((len(win),), 144, device=dev)))
    for key in pipeline.VIDEO_POSE_KEYS:
        pose = dict(bp)
        del pose[key]
        with pytest.raises(RohmB200Error, match=key):
            run(pose, dict(bt))
    with pytest.raises(RohmB200Error, match="windows"):
        run(_take(bp, [0, 1, 2]), dict(bt))
