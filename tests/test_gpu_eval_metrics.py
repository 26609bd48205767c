"""GPU: the evaluation metrics on the device (rohm_b200.metrics) replayed against the reference scripts' own outputs
(tests/golden/eval_metrics.npz, tools/gen_golden.py:gen_eval_metrics), end to end after the video rounds, invariant to
batching and order, and at their edges and refusals."""
import os

import numpy as np
import pytest
import torch

from rohm_b200 import metrics, pipeline
from rohm_b200._lib import RohmB200Error
from test_gpu_noise_streams import _gens
from test_gpu_video_pipeline import _encode, _run, nets  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden", "eval_metrics.npz")
REL = 5e-6
THRESHOLDS = {'speed': 0.1, 'ankle': 0.15, 'toe': 0.1, 'pene': -0.05}


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def close(a, b, rel=REL):
    return np.isnan(b) and np.isnan(a) or abs(a - b) <= rel * abs(b)


def amass_payload(gold, tag):
    G, P = gold[f"{tag}_gt"], gold[f"{tag}_rec"]
    rc, rr = np.zeros(G.shape[:2] + (294,), np.float32), np.zeros(G.shape[:2] + (294,), np.float32)
    rc[..., -4:], rr[..., -4:] = gold[f"{tag}_label_clean"], gold[f"{tag}_label_rec"]
    return {'rec_ric_data_clean_list': G, 'rec_ric_data_rec_list_from_smpl': P, 'motion_repr_clean_list': rc,
            'motion_repr_rec_list': rr}


def video_payloads(gold, dataset):
    out = []
    for r in range(len(gold[f"{dataset}_floor"])):
        p = f"{dataset}_r{r}_"
        d = {'rec_ric_data_rec_list_from_smpl': gold[p + "rec"], 'trans_scene2cano_list': gold[p + "transf"]}
        if dataset == 'egobody':
            d['joints_gt_scene_coord_list'], d['mask_joint_vis_list'] = gold[p + "gt"], gold[p + "mask"]
        out.append(d)
    return out


def own_means_agree(res, per_frame_means):
    for k, v in per_frame_means.items():
        assert close(res[k], v, 1e-12), (k, res[k], v)


@pytest.mark.parametrize("tag", ["amass", "amass_nan"])
def test_amass_replays_the_reference(gold, cuda_device, tag):
    k = 0
    while f"{tag}_run{k}_scheme" in gold:
        run = f"{tag}_run{k}"
        res = metrics.from_payload(amass_payload(gold, tag), str(gold[f"{run}_scheme"]), float(gold[f"{run}_ratio"]),
                                   device=cuda_device)
        f = {n: t.cpu().numpy() for n, t in res['frames'].items()}
        np.testing.assert_array_equal(res['h0'].cpu().numpy(), gold[f"{tag}_h0"])
        for n in ('mpjpe', 'contact_match', 'skating_gt', 'skating_rec', 'accel_error'):
            np.testing.assert_array_equal(f[n], gold[f"{tag}_{n}"], err_msg=n)
        a = res['all']
        for ours, theirs in (('contact_lbl_acc', 'contact_lbl_acc'), ('skating_gt_ratio', 'skating_gt_ratio'),
                             ('skating_rec_ratio', 'skating_rec_ratio'), ('ground_pene_freq', 'pene_freq')):
            assert a[ours] == gold[f"{run}_{theirs}"], (run, ours)
        for ours, theirs in (('mpjpe_global', 'mpjpe_global'), ('mpjpe_global_vis', 'mpjpe_global_vis'),
                             ('mpjpe_global_occ', 'mpjpe_global_occ'), ('accel_error', 'acc_error'),
                             ('ground_pene_dist', 'pene_dist')):
            assert close(a[ours], float(gold[f"{run}_{theirs}"])), (run, ours, a[ours], float(gold[f"{run}_{theirs}"]))
        own_means_agree(a, {'mpjpe_global': f['mpjpe'].astype(np.float64).mean(),
                            'accel_error': f['accel_error'].astype(np.float64).mean(),
                            'ground_pene_dist': f['pene_dist'].astype(np.float64).mean()})
        k += 1


@pytest.mark.parametrize("dataset", ["prox", "egobody"])
def test_video_replays_the_reference(gold, cuda_device, dataset):
    floors = gold[f"{dataset}_floor"]
    res = metrics.from_payload(video_payloads(gold, dataset), dataset=dataset, floor_height=floors, device=cuda_device)
    fr = {n: t.cpu().numpy() for n, t in res['frames'].items()}
    names = [('skating', 'skating_list'), ('acc', 'acc_list'), ('ground_pene_freq', 'ground_pene_freq_list'),
             ('ground_pene_dist', 'ground_pene_dist_list')]
    if dataset == 'egobody':
        names += [('acc_error', 'acc_error_list'), ('gmpjpe', 'gmpjpe_list'), ('mpjpe', 'mpjpe_list')]
    w0, near = 0, 0
    for r in range(len(floors)):
        n = gold[f"{dataset}_r{r}_rec"].shape[0]
        for ours, theirs in names:
            want, got = gold[f"{dataset}_r{r}_{theirs}"], fr[ours][w0:w0 + n]
            if want.dtype == bool:
                np.testing.assert_array_equal(got, want, err_msg=f"{r} {ours}")
            else:
                np.testing.assert_allclose(got, want, rtol=0, atol=1e-6, err_msg=f"{r} {ours}")
        w0 += n
    # the fixture keeps every reference value more than 1e-6 away from a threshold, so decisions are all equal
    for r in range(len(floors)):
        pd = gold[f"{dataset}_r{r}_ground_pene_dist_list"]
        near += int((np.abs(pd - THRESHOLDS['pene']) < 1e-6).sum())
    assert near == 0
    a = res['all']
    assert a['skating'] == gold[f"{dataset}_all_skating"]
    assert a['ground_pene_freq'] == gold[f"{dataset}_all_ground_pene_freq"]
    for k in a:
        if k not in ('skating', 'ground_pene_freq'):
            assert close(a[k], float(gold[f"{dataset}_all_{k}"])), (k, a[k], float(gold[f"{dataset}_all_{k}"]))
    own = {'acc': fr['acc'].astype(np.float64).mean(), 'ground_pene_dist': fr['ground_pene_dist'].astype(np.float64).mean()}
    if dataset == 'egobody':
        own.update(gmpjpe=fr['gmpjpe'].astype(np.float64).mean(), mpjpe=fr['mpjpe'].astype(np.float64).mean())
    own_means_agree(a, own)


def test_video_recordings_alone_batched_and_permuted(gold, cuda_device):
    pl, floors = video_payloads(gold, 'egobody'), gold["egobody_floor"]
    batched = metrics.from_payload(pl, dataset='egobody', floor_height=floors, device=cuda_device)
    perm = np.random.default_rng(0).permutation(len(pl))
    permuted = metrics.from_payload([pl[i] for i in perm], dataset='egobody', floor_height=floors[perm],
                                    device=cuda_device)
    for r in range(len(pl)):
        alone = metrics.from_payload([pl[r]], dataset='egobody', floor_height=floors[r:r + 1], device=cuda_device)
        assert alone['recordings'][0] == batched['recordings'][r] == permuted['recordings'][int(np.flatnonzero(perm == r)[0])]


def test_amass_ragged_equals_each_clip_alone(gold, cuda_device):
    g = np.random.default_rng(3)
    lens = [143, 4100, 7, 2, 300]
    clips = []
    for T in lens:
        G = g.normal(0, 0.5, (T, 22, 3)).astype(np.float32)
        clips.append({'rec_ric_data_clean': G, 'rec_ric_data_rec_from_smpl': (G + g.normal(0, 0.03, G.shape)).astype(np.float32),
                      'motion_repr_clean': g.uniform(0, 1, (T, 294)).astype(np.float32).round(),
                      'motion_repr_rec': g.uniform(0, 1, (T, 294)).astype(np.float32)})
    dev = cuda_device
    ragged = {k: [torch.from_numpy(c[k]).to(dev) for c in clips] for k in clips[0]}
    res = metrics.amass(ragged, 'full', 0.3)
    for b, c in enumerate(clips):
        one = metrics.amass({k: torch.from_numpy(v).to(dev)[None] for k, v in c.items()}, 'full', 0.3)
        assert one['clips'][0] == res['clips'][b] or all(
            (np.isnan(x) and np.isnan(y)) or x == y for x, y in zip(one['clips'][0].values(), res['clips'][b].values()))
        for n, t in one['frames'].items():
            assert torch.equal(t[0], res['frames'][n][b]), n
    assert res['frames']['mpjpe'][1].shape[0] == 4100
    # 'all' pools every clip's frames
    all_mpjpe = np.concatenate([t.cpu().numpy().ravel() for t in res['frames']['mpjpe']]).astype(np.float64)
    assert close(res['all']['mpjpe_global'], all_mpjpe.mean(), 1e-12)


def test_edges_and_refusals(gold, cuda_device):
    dev = cuda_device
    pl = video_payloads(gold, 'prox')[:2]
    empty = {'rec_ric_data_rec_list_from_smpl': np.zeros((0,) + pl[0]['rec_ric_data_rec_list_from_smpl'].shape[1:],
                                                          np.float32), 'trans_scene2cano_list': np.zeros((0, 4, 4), np.float32)}
    res = metrics.from_payload([pl[0], empty, pl[1]], dataset='prox', floor_height=[0.1, 0.2, -0.3], device=dev)
    assert all(np.isnan(v) for v in res['recordings'][1].values())
    assert not np.isnan(res['all']['skating'])
    amass = amass_payload(gold, 'amass')
    assert np.isnan(metrics.from_payload(amass, 'full', 0.0, device=dev)['all']['mpjpe_global_occ'])
    with pytest.raises(RohmB200Error):
        metrics.from_payload(amass, 'upper', device=dev)
    with pytest.raises(RohmB200Error):
        metrics.from_payload(amass, 'full', -0.1, device=dev)
    with pytest.raises(RohmB200Error):
        metrics.from_payload(pl, dataset='h36m', floor_height=[0, 0], device=dev)
    with pytest.raises(RohmB200Error):
        metrics.from_payload(pl, dataset='prox', floor_height=[0.0], device=dev)
    bad = dict(pl[0], trans_scene2cano_list=np.zeros((1, 3, 4), np.float32))
    with pytest.raises(RohmB200Error):
        metrics.from_payload([bad], dataset='prox', floor_height=[0.0], device=dev)
    out = {k: torch.from_numpy(amass[v]).to(dev) for k, v in (('rec_ric_data_clean', 'rec_ric_data_clean_list'),
                                                              ('rec_ric_data_rec_from_smpl', 'rec_ric_data_rec_list_from_smpl'),
                                                              ('motion_repr_clean', 'motion_repr_clean_list'),
                                                              ('motion_repr_rec', 'motion_repr_rec_list'))}
    with pytest.raises(RohmB200Error):
        metrics.amass(dict(out, rec_ric_data_rec_from_smpl=out['rec_ric_data_rec_from_smpl'][:, :10]), 'lower')
    with pytest.raises(RohmB200Error):
        metrics.amass(dict(out, motion_repr_rec=out['motion_repr_rec'][..., :3]), 'lower')


@pytest.mark.parametrize("dataset", ['prox', 'egobody'])
def test_end_to_end_after_the_video_rounds(nets, cuda_device, dataset):  # noqa: F811
    dev = cuda_device
    bt, bp, win = _encode(dataset, nets, dev, with_gt=dataset == 'egobody')
    _, _, _, rec = _run(nets, dev, bt, bp, _gens(dev, [17 + i for i in range(len(win))]))
    floors = [-0.3, 0.1, 0.0]
    res = metrics.video(win, rec, bp, dataset, floors)
    ref = metrics.from_payload(pipeline.video_result_dicts(win, rec, bp), dataset=dataset, floor_height=floors,
                               device=dev)
    assert res['recordings'] == ref['recordings'] and res['all'] == ref['all'] or all(
        (np.isnan(x) and np.isnan(y)) or x == y for a, b in zip(res['recordings'] + [res['all']],
                                                                ref['recordings'] + [ref['all']])
        for x, y in zip(a.values(), b.values()))
    order = res['order'].long()
    for k, t in res['frames'].items():
        assert torch.equal(t[order], ref['frames'][k]), k
    with pytest.raises(RohmB200Error):
        metrics.video(win, rec, bp, dataset, floors[:2])
