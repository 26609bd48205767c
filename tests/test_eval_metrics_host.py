"""CPU checks of the evaluation metrics: the numpy restatement (oracle/metrics_oracle.py) against the reference scripts'
own outputs (tests/golden/eval_metrics.npz), and the kernel's float32 expressions against numpy's."""
import os

import numpy as np
import pytest

from oracle import metrics_oracle as mo

GOLD = os.path.join(os.path.dirname(__file__), "golden", "eval_metrics.npz")
REL = 5e-6  # the reference's float32 np.mean against a float64 mean


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def close(a, b, rel=REL):
    if np.isnan(b):
        return np.isnan(a)
    return abs(a - b) <= rel * abs(b)


@pytest.mark.parametrize("tag", ["amass", "amass_nan"])
def test_oracle_amass_matches_reference(gold, tag):
    f = mo.amass_frames(gold[f"{tag}_gt"], gold[f"{tag}_rec"], gold[f"{tag}_label_clean"], gold[f"{tag}_label_rec"])
    np.testing.assert_array_equal(f['h0'], gold[f"{tag}_h0"])
    for k in ('mpjpe', 'contact_match', 'skating_gt', 'skating_rec', 'accel_error'):
        np.testing.assert_array_equal(f[k], gold[f"{tag}_{k}"], err_msg=k)
    k = 0
    while f"{tag}_run{k}_scheme" in gold:
        run = f"{tag}_run{k}"
        m = mo.amass_metrics(f, str(gold[f"{run}_scheme"]), float(gold[f"{run}_ratio"]))
        for ours, theirs in (('contact_lbl_acc', 'contact_lbl_acc'), ('skating_gt_ratio', 'skating_gt_ratio'),
                             ('skating_rec_ratio', 'skating_rec_ratio'), ('ground_pene_freq', 'pene_freq')):
            assert m[ours] == gold[f"{run}_{theirs}"], (run, ours)  # ratios of counts: bit-equal
        for ours, theirs in (('mpjpe_global', 'mpjpe_global'), ('mpjpe_global_vis', 'mpjpe_global_vis'),
                             ('mpjpe_global_occ', 'mpjpe_global_occ'), ('accel_error', 'acc_error'),
                             ('ground_pene_dist', 'pene_dist')):
            assert close(m[ours], float(gold[f"{run}_{theirs}"])), (run, ours, m[ours], float(gold[f"{run}_{theirs}"]))
        k += 1
    assert k >= 1


def test_amass_fixture_covers_the_edges(gold):
    assert np.isnan(gold["amass_nan_h0"][0]) and not np.isnan(gold["amass_nan_h0"][1])
    assert np.isnan(gold["amass_run2_mpjpe_global_occ"])  # 'full' at ratio 0: empty occluded set
    assert str(gold["amass_run3_scheme"]) == 'full' and float(gold["amass_run3_ratio"]) == 0.7
    assert gold["amass_skating_gt"].any() and gold["amass_skating_rec"].any()
    assert (gold["amass_gt"][..., [7, 10, 8, 11], 2] == np.float32(0.1)).any()


@pytest.mark.parametrize("dataset", ["prox", "egobody"])
def test_oracle_video_matches_reference(gold, dataset):
    floors = gold[f"{dataset}_floor"]
    per = []
    for r in range(len(floors)):
        p = f"{dataset}_r{r}_"
        f = mo.video_frames(gold[p + "rec"], gold[p + "transf"], dataset, float(floors[r]),
                            gold.get(p + "gt"), gold.get(p + "mask"))
        per.append(f)
        pairs = [('skating', 'skating_list'), ('acc', 'acc_list'), ('ground_pene_freq', 'ground_pene_freq_list'),
                 ('ground_pene_dist', 'ground_pene_dist_list')]
        if dataset == 'egobody':
            pairs += [('acc_error', 'acc_error_list'), ('gmpjpe', 'gmpjpe_list'), ('mpjpe', 'mpjpe_list'),
                      ('mpjpe_vis', 'mpjpe_list_vis'), ('mpjpe_occ', 'mpjpe_list_occ')]
        for ours, theirs in pairs:
            np.testing.assert_array_equal(f[ours], gold[p + theirs], err_msg=f"{r} {ours}")
    all_, _ = mo.video_metrics(per)
    for k, v in all_.items():
        ref = float(gold[f"{dataset}_all_{k}"])
        assert (v == ref) if k in ('skating', 'ground_pene_freq') else close(v, ref), (k, v, ref)


def _edge_floats(g, n):
    x = g.standard_normal(n).astype(np.float32) * np.float32(10) ** g.integers(-20, 20, n).astype(np.float32)
    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 1e-40, 3e38, -3e38], np.float32)
    idx = g.integers(0, n, n // 20)
    x[idx] = special[g.integers(0, len(special), len(idx))]
    sub = g.integers(0, n, n // 20)
    x[sub] = (g.standard_normal(len(sub)) * 1e-39).astype(np.float32)
    return x


def test_kernel_expressions_match_numpy():
    """norm / acceleration / joint-mean in the kernel's explicit order against numpy's own evaluation, >= 1e6 inputs."""
    g = np.random.default_rng(5)
    with np.errstate(all='ignore'):
        x = _edge_floats(g, 3 * 400000).reshape(-1, 3)
        np.testing.assert_array_equal(mo.norm3(x), np.linalg.norm(x, axis=-1))
        y = _edge_floats(g, 2 * 500000).reshape(-1, 2)
        np.testing.assert_array_equal(mo.norm2(y), np.linalg.norm(y, axis=-1))
        z = _edge_floats(g, 3 * 400000).reshape(-1, 3, 1).transpose(1, 0, 2)  # [3 frames, n, 1]
        seq = np.ascontiguousarray(z.transpose(1, 0, 2))  # [n, 3, 1]: frames along axis 1
        fps = 30
        ref = (seq[:, 2:] - 2 * seq[:, 1:-1] + seq[:, :-2]) * (fps ** 2)
        np.testing.assert_array_equal(mo.accel(seq), ref)
        v = _edge_floats(g, 22 * 60000).reshape(-1, 22)
        np.testing.assert_array_equal(mo.mean22(v), v.mean(axis=-1))
