"""The evaluation-metric kernels (csrc/metrics.cu through rohm_b200.metrics) against the numpy restatement
(oracle/metrics_oracle.py) at the inputs where a comparison operator, a summation order or a stride goes wrong: every
skating, height, penetration and contact threshold hit exactly and one float32 ulp either side, clip lengths around the
kernel's 128-thread frame stride and the t + 1 < T / t + 2 < T edges, subnormals, +-0, +-inf, NaN and 3e38 in the
joints, the occlusion windows clamped to short clips, ground truth and masks longer than the windows, transforms whose
inverse needs a row exchange, and the cross-clip reduction over permuted, empty and many groups.

Tolerances, and where they come from:
- Per-frame values are compared bit for bit (``assert_bits``: equal float32 bit patterns, any NaN matching any NaN).
  The sign of a zero counts: the penetration clamp maps d = -0.0 to +0.0 as numpy's ``pd[pd >= 0] = 0`` does.
- Counts and ratios of counts are compared with ``==``: both are integers, or the same float64 division of them.
- A float64 sum of n float32 values, in the kernel's order, against the exactly rounded ``math.fsum``: any order of
  the n - 1 additions lies within gamma_{n-1} * sum|x| of the exact sum, gamma_k = k u / (1 - k u), u = 2^-53 (Higham,
  Accuracy and Stability of Numerical Algorithms, 2nd ed., (4.4)); the kernel's additions of 0.0 are exact.
- ``rohm_eval_reduce`` adds the items of a group one by one in the given order and the groups in order, so a float64
  loop in that order reproduces it bit for bit.
- Scene coordinates under a general rigid transform: see ``test_video_general_transforms_within_the_derived_bound``.
"""
import math

import numpy as np
import pytest
import torch

from oracle import metrics_oracle as mo
from rohm_b200 import metrics
from test_eval_metrics_host import _edge_floats

F32 = np.float32
U32, U64 = 2.0 ** -24, 2.0 ** -53
LENGTHS = (1, 2, 3, 4, 64, 65, 127, 128, 129, 130, 255, 256, 257, 4999)
SCHEMES = (('lower', 0.0), ('full', 0.0), ('full', 0.3), ('full', 0.7), ('full', 1.0), ('full', 1e10))
WIDTH = 9  # motion-representation channels: the contact labels are the last 4, the first 5 are noise to skip
DX = F32(F32(0.1) / F32(30))  # fl(fl(sqrt(fl(DX^2))) * 30) == float32(0.1): a foot step exactly at the speed threshold
FLOORS = (0.0, 0.25, -1.5)
DATASETS = {'prox': (2, (0, 1)), 'egobody': (1, (0, 2))}  # up axis, horizontal axes


def around(x):
    """float32(x) and its neighbours one ulp below and above."""
    x = F32(x)
    return [np.nextafter(x, F32(-np.inf)), x, np.nextafter(x, F32(np.inf))]


CLEAN_LABELS = np.array([0, 1, 0.3, 0.5, np.nan], F32)
REC_LABELS = np.array(around(0.5) + [0, 1, 0.7, np.nan, np.inf, -np.inf], F32)
PENE = np.array(around(-0.05) + [-0.0, 0.0, -1.0], F32)


def assert_bits(got, want, msg=''):
    """Equal bit patterns (bools: equal values); a NaN matches any NaN, whose payload numpy and CUDA choose apart."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (msg, got.shape, want.shape)
    if want.dtype == bool:
        np.testing.assert_array_equal(got, want, err_msg=msg)
        return
    if want.dtype == np.float64:  # the oracle's float64 mean of two toes' 0 / 1: exact in float32
        assert (want.astype(F32) == want).all(), msg
        want = want.astype(F32)
    assert got.dtype == want.dtype == F32, (msg, got.dtype, want.dtype)
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    if not same.all():
        i = tuple(np.argwhere(~same)[0])
        pytest.fail(f"{msg}: {(~same).sum()} of {same.size} differ, first at {i}: {got[i]!r} vs {want[i]!r}")


def assert_sum(got, values, msg=''):
    """got: a float64 sum of `values` in some order of n - 1 additions -> within gamma_{n-1} sum|x| of math.fsum."""
    v = np.asarray(values, np.float64).ravel()
    if np.isnan(v).any() or (np.isposinf(v).any() and np.isneginf(v).any()):
        assert np.isnan(got), (msg, got)
        return
    if np.isinf(v).any():
        assert got == v[np.isinf(v)][0], (msg, got)
        return
    k = max(v.size - 1, 0)
    tol = k * U64 / (1 - k * U64) * math.fsum(np.abs(v))
    assert abs(got - math.fsum(v)) <= tol, (msg, got, math.fsum(v), tol)


def same(a, b):
    return (np.isnan(a) and np.isnan(b)) or a == b


def spy(monkeypatch, name):
    """The raw (sums, counts) rows metrics.<name> turns into a result dict, in call order."""
    rows, real = [], getattr(metrics, name)
    monkeypatch.setattr(metrics, name, lambda *a: rows.append(a) or real(*a))
    return rows


# ----------------------------------------------------------------------------------------------------- input builders
def tie_joints(g, T, up=2, horiz=(0, 1), floor=0.0, penetrate=False):
    """[T,22,3] float32 joints whose feet step and stand on the skating thresholds over `floor`, or one ulp beside them,
    while the rest of the skating rule holds; with `penetrate` the toes also sink to -0.05, one ulp beside it, and
    to -0.0.  The feet sit at 0 on even frames and at a step on odd ones, so every frame pair moves by the step
    exactly (the difference with 0 is exact); other joints stand 0.5 m or more over the floor."""
    fl = F32(floor)
    lift = lambda h: (h if floor == 0 else fl + h).astype(F32)  # 0 + -0.0 would lose the sign of a zero
    X = np.zeros((T, 22, 3), F32)
    X[..., list(horiz)] = g.normal(0, 0.3, (T, 22, 2))
    X[..., up] = lift(F32(0.5) + np.abs(g.normal(0, 0.3, (T, 22))).astype(F32))
    step = np.zeros((T, 4), F32)
    axis = np.zeros(T, int)
    for t in range(1, T, 2):
        step[t] = 0.05  # 1.5 m/s
        k = g.integers(0, 4)
        if k == 1:
            step[t, g.integers(0, 4)] = g.choice(around(DX))
        elif k == 2:
            step[t] = g.choice(around(DX))
        elif k == 3:
            step[t] = 0
        axis[t] = g.integers(0, 2)
    hts = np.empty((T, 4), F32)
    hts[:, [0, 2]], hts[:, [1, 3]] = 0.05, 0.02  # FOOT order: ankle, toe, ankle, toe
    for t in range(T):
        k = g.integers(0, 3)
        f = int(g.integers(0, 4))
        if k == 0:
            hts[t, f] = g.choice(around(0.15 if f % 2 == 0 else 0.1))
        elif k == 1 and penetrate:
            hts[t, 1 + 2 * (f % 2)] = g.choice(PENE)
    for f, j in enumerate(mo.FOOT):
        X[:, j, list(horiz)] = 0
        X[np.arange(T), j, np.asarray(horiz)[axis]] = step[:, f]
        X[:, j, up] = lift(hts[:, f])
    return X


def amass_clip(g, T, kind):
    """One clip {G, P, label_clean, label_rec, repr_clean, repr_rec} of a kind:
    'ties'  the thresholds of tie_joints on G and P with the clean clip's lowest z exactly +0.0, contact labels at
            0.5 and beside it, NaN and +-inf, clean labels 0.3, 0.5 and NaN besides 0 and 1;
    'edge'  a random walk with a tenth of G and P replaced by _edge_floats (subnormals, +-0, +-inf, NaN, 3e38) and
            one NaN in P, labels likewise;
    'nan_z' a random walk with one NaN clean z (h0 NaN: neither G nor P skates) and NaN / inf labels;
    'plain' a random walk."""
    if kind == 'ties':
        G = tie_joints(g, T)
        G[0, 0, 2] = 0.0
        P = tie_joints(g, T, penetrate=True)
        lc, lr = g.choice(CLEAN_LABELS, (T, 4)), g.choice(REC_LABELS, (T, 4))
    else:
        G = (g.normal(0, 0.02, (T, 22, 3)).cumsum(0) + g.normal(0, 0.3, (1, 22, 3))).astype(F32)
        P = (G + g.normal(0, 0.03, G.shape)).astype(F32)
        lc, lr = g.integers(0, 2, (T, 4)).astype(F32), g.uniform(0, 1, (T, 4)).astype(F32)
        if kind == 'edge':
            for X in (G, P, lc, lr):
                x = X.reshape(-1)
                hit = g.random(x.size) < 0.1
                x[hit] = _edge_floats(g, x.size)[hit]
            P[g.integers(0, T), g.integers(0, 22), 0] = np.nan
        elif kind == 'nan_z':
            G[g.integers(0, T), g.integers(0, 22), 2] = np.nan
            lr[g.integers(0, T), g.integers(0, 4)] = np.nan
            lr[g.integers(0, T), g.integers(0, 4)] = np.inf
            lc[g.integers(0, T), g.integers(0, 4)] = np.nan
    rc, rr = g.normal(0, 1, (T, WIDTH)).astype(F32), g.normal(0, 1, (T, WIDTH)).astype(F32)
    rc[:, -4:], rr[:, -4:] = lc, lr
    return {'G': G, 'P': P, 'lc': lc, 'lr': lr, 'rc': rc, 'rr': rr}


def amass_payload(clips, ragged):
    keys = (('rec_ric_data_clean_list', 'G'), ('rec_ric_data_rec_list_from_smpl', 'P'),
            ('motion_repr_clean_list', 'rc'), ('motion_repr_rec_list', 'rr'))
    if ragged:
        return {k: [c[v] for c in clips] for k, v in keys}
    return {k: np.stack([c[v] for c in clips]) for k, v in keys}


def signed_perms(g, n, zero_diag=False):
    """n random 3x3 signed permutation matrices; zero_diag: each with R[0,0] == 0, so Gauss-Jordan must exchange
    rows at its first column."""
    out = []
    while len(out) < n:
        p = g.permutation(3)
        if zero_diag and p[0] == 0:
            continue
        R = np.zeros((3, 3), F32)
        R[np.arange(3), p] = g.choice([-1, 1], 3)
        out.append(R)
    return out


def transform(R, t):
    A = np.eye(4, dtype=F32)
    A[:3, :3], A[:3, 3] = R, t
    return A


def video_windows(g, T, dataset):
    """Three recordings on FLOORS, three windows each, interleaved in the batch (window 3i + r is recording r's i-th):
    0: the ties of tie_joints over the recording's floor in the scene, transf a signed permutation with a zero
       diagonal and no translation (scene -> canonical -> scene is exact);
    1: the same under any signed permutation;
    2: random canonical joints under a signed permutation and a dyadic translation.
    Ground truth and mask_joint_vis hold 7 more frames than T (noise there); the mask takes 0, 1, 0.25 and 0.5."""
    up, horiz = DATASETS[dataset]
    R_, W = len(FLOORS), 3 * len(FLOORS)
    rec, transf = np.empty((W, T, 22, 3), F32), np.empty((W, 4, 4), F32)
    gt = g.normal(0, 2, (W, T + 7, 22, 3)).astype(F32)
    mask = g.choice(np.array([0, 1, 0.25, 0.5], F32), (W, T + 7, 22))
    for r, fl in enumerate(FLOORS):
        for i in range(3):
            w = 3 * i + r
            R = signed_perms(g, 1, zero_diag=i == 0)[0]
            if i < 2:
                S = tie_joints(g, T, up, horiz, fl, penetrate=True)
                rec[w] = S @ R.T  # one +-1 per row: exact
                transf[w] = transform(R, 0)
                gt[w, :T] = S + g.normal(0, 0.05, S.shape).astype(F32)
            else:
                rec[w] = g.normal(0, 0.02, (T, 22, 3)).cumsum(0) + g.normal(0, 0.3, (1, 22, 3))
                transf[w] = transform(R, g.integers(-160, 161, 3) / 16)
    win_rec = np.tile(np.arange(R_, dtype=np.int32), 3)
    order = np.concatenate([np.arange(r, W, R_) for r in range(R_)]).astype(np.int32)
    return rec, transf, gt, mask, win_rec, order


def run_video(dev, rec, transf, gt, mask, win_rec, order, dataset):
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev) if a is not None else None
    n_per_rec = np.bincount(win_rec, minlength=len(FLOORS)).tolist()
    return metrics._video(up(rec), up(transf), up(gt), up(mask), up(win_rec), up(order), n_per_rec, dataset,
                          np.array(FLOORS))


def foot_state(X, base, up, horiz):
    """The oracle's per-pair foot speeds v [T-1,4] and heights over `base` h [T-1,4] of joints X [T,22,3]."""
    f = X[:, mo.FOOT]
    v = (mo.norm2(f[1:][..., list(horiz)] - f[:-1][..., list(horiz)]) * F32(30)).astype(F32)
    return v, (f[:-1, :, up] - F32(base)).astype(F32)


def skating_rule(v, h, speed=np.greater, ankle=np.less, toe=np.less):
    side = lambda a, b: (speed(v[:, a], F32(0.1)) & speed(v[:, b], F32(0.1)) & ankle(h[:, a], F32(0.15)) &
                         toe(h[:, b], F32(0.1)))
    return side(0, 1) & side(2, 3)


def decisive_ties(v, h):
    """Which of the skating rule's comparisons decide some frame pair on their threshold: the rule with that
    comparison made inclusive gives another answer there."""
    base = skating_rule(v, h)
    return {'speed': (skating_rule(v, h, speed=np.greater_equal) != base).any(),
            'ankle': (skating_rule(v, h, ankle=np.less_equal) != base).any(),
            'toe': (skating_rule(v, h, toe=np.less_equal) != base).any()}


# ------------------------------------------------------------------------------------- the constructions (no GPU)
def test_constructed_inputs_hit_the_thresholds():
    """The tie builders put the oracle's own values on every threshold, deciding frame pairs there; without this the
    bit-for-bit tests below could pass with a flipped comparison."""
    g = np.random.default_rng(11)
    with np.errstate(all='ignore'):
        c = amass_clip(g, 300, 'ties')
        f = mo.amass_frames(c['G'][None], c['P'][None], c['lc'][None], c['lr'][None])
        assert f['h0'][0] == 0 and not np.signbit(f['h0'][0])
        for X in (c['G'], c['P']):
            v, h = foot_state(X, 0.0, 2, (0, 1))
            assert (v == F32(0.1)).any() and (h[:, [0, 2]] == F32(0.15)).any() and (h[:, [1, 3]] == F32(0.1)).any()
            assert all(decisive_ties(v, h).values())
        v, h = foot_state(c['G'], 0.0, 2, (0, 1))
        np.testing.assert_array_equal(skating_rule(v, h), f['skating_gt'][0])
        d = c['P'][:, [10, 11], 2]
        assert (d == F32(-0.05)).any() and (d == np.nextafter(F32(-0.05), F32(0))).any()
        negzero = lambda a: np.signbit(a) & (a == 0)
        assert negzero(d).any() and not negzero(f['pene_dist']).any()  # -0.0 clamped to +0.0
        assert (c['lr'] == F32(0.5)).any() and np.isnan(c['lr']).any() and np.isinf(c['lr']).any()
        nz = amass_clip(g, 300, 'nan_z')
        fz = mo.amass_frames(nz['G'][None], nz['P'][None], nz['lc'][None], nz['lr'][None])
        assert np.isnan(fz['h0'][0]) and not fz['skating_gt'].any() and not fz['skating_rec'].any()
        edge = amass_clip(g, 300, 'edge')
        x = np.concatenate([edge['G'].ravel(), edge['P'].ravel()])
        assert np.isnan(x).any() and np.isinf(x).any() and ((x != 0) & (np.abs(x) < 1.2e-38)).any()
        assert (np.abs(x) > 1e38).any()

        for dataset, (up, horiz) in DATASETS.items():
            rec, transf, _, _, win_rec, _ = video_windows(np.random.default_rng(12), 300, dataset)
            for w in range(len(transf)):
                exact = transform(transf[w, :3, :3].T, -transf[w, :3, :3].T @ transf[w, :3, 3])
                assert (np.linalg.inv(transf[w]) == exact).all()
            assert (transf[:len(FLOORS), 0, 0] == 0).all()
            for r, fl in enumerate(FLOORS):
                ties = {'speed': False, 'ankle': False, 'toe': False}
                pene = False
                for w in (r, r + 3):
                    S = mo.scene_joints(rec[w:w + 1], transf[w:w + 1])[0]
                    v, h = foot_state(S, fl, up, horiz)
                    ties = {k: ties[k] or t for k, t in decisive_ties(v, h).items()}
                    pene |= ((S[:, [10, 11], up] - F32(fl)).astype(F32) == F32(-0.05)).any()
                # over a floor of 0.25 no float32 lies exactly 0.1 or -0.05 above it, over -1.5 none lies 0.15, 0.1 or
                # -0.05 above it; the neighbours one ulp either side still straddle the threshold
                want = {0.0: (True, True, True, True), 0.25: (True, True, False, False),
                        -1.5: (True, False, False, False)}[fl]
                assert (ties['speed'], ties['ankle'], ties['toe'], pene) == want, (dataset, fl, ties, pene)


# ------------------------------------------------------------------------------------------------------ AMASS
def check_amass(res, rows, clips, scheme, ratio, frames_too=True):
    """res / rows (the spied _amass_values rows: per clip, then 'all') against the oracle run on each clip alone."""
    B = len(clips)
    assert len(rows) == B + 1
    all_vals = {k: [] for k in ('mpjpe', 'vis', 'occ', 'accel', 'pene')}
    all_counts = np.zeros(11, np.int64)
    for b, c in enumerate(clips):
        T = c['G'].shape[0]
        with np.errstate(all='ignore'):
            f = {k: v[0] for k, v in mo.amass_frames(c['G'][None], c['P'][None], c['lc'][None], c['lr'][None]).items()}
        if frames_too:
            assert_bits(res['h0'].cpu().numpy()[b], f['h0'], f"clip {b} (T={T}) h0")
            for k in ('mpjpe', 'accel_error', 'skating_gt', 'skating_rec', 'contact_match', 'pene_freq', 'pene_dist'):
                assert_bits(res['frames'][k][b].cpu().numpy(), f[k], f"clip {b} (T={T}) {k}")
        occ = np.zeros((T, 22), bool)
        if scheme == 'lower':
            occ[:, mo.LOWER_OCCLUDED] = True
        else:
            occ[65:65 + int(ratio * 145)] = True
        e = f['mpjpe']
        vals = {'mpjpe': e, 'vis': e[~occ], 'occ': e[occ], 'accel': f['accel_error'], 'pene': f['pene_dist']}
        want_c = np.array([T * 22, (~occ).sum(), occ.sum(), f['contact_match'].sum(), 4 * T, f['skating_gt'].sum(),
                           f['skating_rec'].sum(), max(T - 1, 0), max(T - 2, 0) * 22, f['pene_freq'].sum(), 2 * T])
        s, cnt = rows[b]
        np.testing.assert_array_equal(cnt, want_c, err_msg=f"clip {b} (T={T}) counts")
        for i, k in enumerate(vals):
            assert_sum(s[i], vals[k], f"clip {b} (T={T}) sum {k}")
            all_vals[k].append(vals[k].ravel())
        all_counts += want_c
        m = res['clips'][b]
        div = lambda a, n: a / n if n else np.nan
        for k, (num, den) in {'contact_lbl_acc': (3, 4), 'skating_gt_ratio': (5, 7), 'skating_rec_ratio': (6, 7),
                              'ground_pene_freq': (9, 10)}.items():
            assert same(m[k], div(float(want_c[num]), float(want_c[den]))), (b, T, k)
        if not occ.any():
            assert np.isnan(m['mpjpe_global_occ']), (b, T)
        if np.isnan(e).any():
            assert np.isnan(m['mpjpe_global']), (b, T)
    s, cnt = rows[B]
    np.testing.assert_array_equal(cnt, all_counts, err_msg="'all' counts")
    for i, k in enumerate(all_vals):
        assert_sum(s[i], np.concatenate(all_vals[k]), f"'all' sum {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("T", LENGTHS)
def test_amass_batched_lengths_bit_for_bit(cuda_device, monkeypatch, T):
    """[B,T,...] batches of the four clip kinds: per-frame arrays bit for bit, counts exact, sums within gamma_{n-1};
    the NaN clips' means are NaN, their neighbours' finite, 'all' NaN."""
    g = np.random.default_rng(100 + T)
    kinds = ('ties', 'edge', 'nan_z', 'plain')
    clips = [amass_clip(g, T, k) for k in kinds]
    scheme, ratio = SCHEMES[LENGTHS.index(T) % len(SCHEMES)]
    rows = spy(monkeypatch, '_amass_values')
    res = metrics.from_payload(amass_payload(clips, ragged=False), scheme, ratio, device=cuda_device)
    check_amass(res, [(np.array(s), np.array(c)) for s, c in rows], clips, scheme, ratio)
    finite = [np.isfinite(res['clips'][b]['mpjpe_global']) for b in range(len(kinds))]
    assert finite == [True, False, False, True]
    assert np.isnan(res['all']['mpjpe_global'])


@pytest.mark.gpu
def test_amass_ragged_lengths_and_occlusion_bit_for_bit(cuda_device, monkeypatch):
    """One ragged batch mixing every length (and 100, which ends inside [65, 108) of 'full' at 0.3) and every clip
    kind, under every occlusion scheme: each clip against the oracle run on that clip alone, occluded and visible
    counts from an explicit mask per clip, 'full' at 1e10 clamped to 2^31 - 1 and then to each clip."""
    g = np.random.default_rng(7)
    kinds = ('ties', 'edge', 'nan_z', 'plain')
    clips = [amass_clip(g, T, kinds[i % 4]) for i, T in enumerate(LENGTHS + (100,) + LENGTHS[::-1])]
    rows = spy(monkeypatch, '_amass_values')
    for n, (scheme, ratio) in enumerate(SCHEMES):
        rows.clear()
        res = metrics.from_payload(amass_payload(clips, ragged=True), scheme, ratio, device=cuda_device)
        check_amass(res, [(np.array(s), np.array(c)) for s, c in rows], clips, scheme, ratio, frames_too=n == 0)


# ------------------------------------------------------------------------------------------------------ video
def check_video(res, rows, rec, transf, gt, mask, win_rec, order, dataset):
    """Per recording: the oracle's per-window arrays bit for bit, the skating count exact, the sums within gamma."""
    with_gt = gt is not None
    R = len(FLOORS)
    assert len(rows) == R + 1
    fr = {k: t.cpu().numpy() for k, t in res['frames'].items()}
    keys = ('skating', 'acc', 'ground_pene_freq', 'ground_pene_dist') + (
        ('acc_error', 'gmpjpe', 'mpjpe') if with_gt else ())
    cat = {k: [] for k in ('skating', 'acc', 'acc_error', 'gmpjpe', 'mpjpe', 'vis_num', 'vis_den', 'occ_num',
                           'occ_den', 'pene_freq', 'pene_dist')}
    for r in range(R):
        idx = order[np.flatnonzero(win_rec[order] == r)]
        with np.errstate(all='ignore'):
            want = mo.video_frames(rec[idx], transf[idx], dataset, FLOORS[r], gt[idx] if with_gt else None,
                                   mask[idx] if with_gt else None)
        for k in keys:
            assert_bits(fr[k][idx], want[k], f"{dataset} recording {r} {k}")
        vals = {'skating': want['skating'], 'acc': want['acc'], 'pene_freq': want['ground_pene_freq'],
                'pene_dist': want['ground_pene_dist']}
        if with_gt:
            m = want['joint_mask']
            vals.update(acc_error=want['acc_error'], gmpjpe=want['gmpjpe'], mpjpe=want['mpjpe'],
                        vis_num=want['mpjpe_vis'], vis_den=m, occ_num=want['mpjpe_occ'], occ_den=F32(1) - m)
        s, sk = rows[r][0], rows[r][1]
        assert sk == want['skating'].sum(), (r, sk)
        for i, k in enumerate(metrics.VIDEO_SUMS):
            if k in vals:
                assert_sum(s[i], vals[k], f"{dataset} recording {r} sum {k}")
        for k, v in vals.items():
            cat[k].append(np.ravel(v))
        out = res['recordings'][r]
        assert out['skating'] == want['skating'].sum() / want['skating'].size
        pf = want['ground_pene_freq'].astype(np.float64)
        assert out['ground_pene_freq'] == pf.sum() / pf.size
    s, sk = rows[R][0], rows[R][1]
    assert sk == np.concatenate(cat['skating']).sum()
    for i, k in enumerate(metrics.VIDEO_SUMS):
        if cat[k]:
            assert_sum(s[i], np.concatenate(cat[k]), f"{dataset} 'all' sum {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("dataset", tuple(DATASETS))
@pytest.mark.parametrize("T", (3, 4, 129, 145, 300))
def test_video_exact_transforms_bit_for_bit(cuda_device, monkeypatch, dataset, T):
    """Signed-permutation transforms (zero diagonals among them) with dyadic translations: the float32 inverse is
    exact and each coordinate's FMA chain has one non-zero product, so the kernel's scene joints are numpy's whatever
    the BLAS, and every per-frame value is the oracle's bit for bit, thresholds over floors 0, 0.25 and -1.5
    included.  Ground truth and masks are 7 frames longer than the windows; recordings are interleaved in the batch.
    For PROX the pass without ground truth is checked too."""
    g = np.random.default_rng(1000 * T + len(dataset))
    rec, transf, gt, mask, win_rec, order = video_windows(g, T, dataset)
    rows = spy(monkeypatch, '_video_values')
    res = run_video(cuda_device, rec, transf, gt, mask, win_rec, order, dataset)
    check_video(res, [(np.array(r[0]), r[1]) for r in rows], rec, transf, gt, mask, win_rec, order, dataset)
    if dataset == 'prox':
        rows.clear()
        res = run_video(cuda_device, rec, transf, None, None, win_rec, order, dataset)
        check_video(res, [(np.array(r[0]), r[1]) for r in rows], rec, transf, None, None, win_rec, order, dataset)


def rotation(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + math.sin(angle) * K + (1 - math.cos(angle)) * K @ K


@pytest.mark.gpu
def test_video_general_transforms_within_the_derived_bound(cuda_device):
    """Random rotations, rotations within 1e-4 rad of 180 degrees (some about axes that leave a diagonal entry near
    zero), translations up to 1e3 m.  Reference: the scene joints in float64 from the float64 inverse of the float32
    matrix, S = M x + t, and gmpjpe_ref = ||g - S||.

    Bound.  Per coordinate the kernel computes fl(fma(x2, m2, fma(x1, m1, fl(x0 m0))) + t) from m, t = M, t rounded to
    float32 (one rounding, u = 2^-24, on each entry): four roundings on the x0 term, fewer on the others, so
    |S_kernel,i - S_i| <= (gamma_4 + u (1 + gamma_4)) A_i = (5u + O(u^2)) A_i with A_i = sum_k |M_ik||x_k| + |t_i|.
    The float64 inverses (the kernel's Gauss-Jordan and LAPACK's) differ from the exact one by a few 2^-53 relative
    for these orthogonal blocks, 2^-29 of u.  c = 6 covers the second-order terms and both: E = c u ||A||_2 bounds
    the scene joint's error.  gmpjpe is norm3 of fl(g - S_kernel) in float32: the difference, the squares, two adds and
    the square root give at most 3.5u relative, 4u with second-order terms.  So
    |gmpjpe - gmpjpe_ref| <= E + 4u (gmpjpe_ref + E)."""
    g = np.random.default_rng(21)
    T, W, c = 145, 12, 6.0
    Rs = []
    for w in range(W):
        if w < 4:
            q = g.normal(size=4)
            Rs.append(rotation(q[:3], 2 * math.atan2(np.linalg.norm(q[:3]), q[3])))
        else:
            axis = g.normal(size=3) if w < 8 else [1, 1, 0] if w % 2 else [0, 1, -1]
            Rs.append(rotation(axis, math.pi - g.uniform(0, 1e-4)))
    scale = np.where(np.arange(W) % 2 == 0, 1.0, 1e3)
    transf = np.stack([transform(R.astype(F32), g.uniform(-1, 1, 3) * s) for R, s in zip(Rs, scale)]).astype(F32)
    rec = g.normal(0, 1, (W, T, 22, 3)).astype(F32)
    inv = np.linalg.inv(transf.astype(np.float64))
    M, t = inv[:, None, None, :3, :3], inv[:, None, None, :3, 3]
    S = (M @ rec.astype(np.float64)[..., None])[..., 0] + t
    gt = (S + g.normal(0, 0.05, S.shape)).astype(F32)
    mask = np.ones((W, T, 22), F32)
    win_rec = (np.arange(W) % 3).astype(np.int32)
    order = np.concatenate([np.flatnonzero(win_rec == r) for r in range(3)]).astype(np.int32)
    res = run_video(cuda_device, rec, transf, gt, mask, win_rec, order, 'prox')
    got = res['frames']['gmpjpe'].cpu().numpy().astype(np.float64)
    ref = np.linalg.norm(gt.astype(np.float64) - S, axis=-1)
    A = (np.abs(M) @ np.abs(rec.astype(np.float64))[..., None])[..., 0] + np.abs(t)
    E = c * U32 * np.linalg.norm(A, axis=-1)
    tol = E + 4 * U32 * (ref + E)
    err = np.abs(got - ref)
    assert (err <= tol).all(), (float((err / tol).max()), np.unravel_index(np.argmax(err / tol), err.shape))


@pytest.mark.gpu
def test_video_bad_transforms_stay_in_their_window(cuda_device, monkeypatch):
    """A singular transf (zero rotation block) and one holding a NaN give non-finite values in their own windows and
    NaN for their recording and 'all'; every other window and recording is bit-identical to a run with good
    transforms in their place."""
    g = np.random.default_rng(31)
    rec, transf, gt, mask, win_rec, order = video_windows(g, 129, 'egobody')
    bad = transf.copy()
    bad[1, :3, :3] = 0  # recording 1
    bad[4, 1, 2] = np.nan  # recording 1
    rows = spy(monkeypatch, '_video_values')
    good = run_video(cuda_device, rec, transf, gt, mask, win_rec, order, 'egobody')
    good_rows = [np.array(r[0]) for r in rows]
    rows.clear()
    res = run_video(cuda_device, rec, bad, gt, mask, win_rec, order, 'egobody')
    keep = np.flatnonzero(win_rec != 1)
    for k, t in res['frames'].items():
        assert_bits(t.cpu().numpy()[keep], good['frames'][k].cpu().numpy()[keep], k)
    for w in (1, 4):
        assert not np.isfinite(res['frames']['gmpjpe'][w].cpu().numpy()).all(), w
    for r in (0, 2):
        np.testing.assert_array_equal(np.array(rows[r][0]).view(np.int64), good_rows[r].view(np.int64), str(r))
        assert all(same(res['recordings'][r][k], v) for k, v in good['recordings'][r].items()), r
    assert np.isnan(res['recordings'][1]['gmpjpe']) and np.isnan(res['all']['gmpjpe'])


# ------------------------------------------------------------------------------------------------------ reduce
def reduce_expected(sums, counts, order, off):
    G = len(off) - 1
    out_s, out_c = np.zeros((G + 1, sums.shape[1])), np.zeros((G + 1, counts.shape[1]), np.int64)
    for q in range(G):
        a, c = np.zeros(sums.shape[1]), np.zeros(counts.shape[1], np.int64)
        for i in range(off[q], off[q + 1]):
            a = a + sums[order[i]]  # elementwise float64 additions, one item at a time
            c = c + counts[order[i]]
        out_s[q], out_c[q] = a, c
        out_s[G], out_c[G] = out_s[G] + a, out_c[G] + c
    return out_s, out_c


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ['permuted', 'no_groups', 'thousand'])
def test_reduce_bit_for_bit(cuda_device, layout):
    """rohm_eval_reduce against the float64 loop in its order, bit for bit, with 40 + 9 columns (two 32-thread
    blocks): a permuted order whose groups hold 0, 1 and many items and leave the last items out; no groups; 1000
    groups over 3000 items.  Sums span 24 decades, so another order would change bits."""
    g = np.random.default_rng(41)
    ks, kc = 40, 9
    N = 3000 if layout == 'thousand' else 60
    sums = g.standard_normal((N, ks)) * 10.0 ** g.integers(-12, 12, (N, ks))
    counts = g.integers(-2 ** 40, 2 ** 40, (N, kc))
    order = g.permutation(N).astype(np.int32)
    if layout == 'no_groups':
        off = np.zeros(1, np.int32)
    elif layout == 'thousand':
        off = np.concatenate([[0], np.sort(g.integers(0, N + 1, 999)), [N]]).astype(np.int32)
        assert (np.diff(off) == 0).any() and (np.diff(off) == 1).any()
    else:
        off = np.array([0, 0, 1, 30, 30, 55], np.int32)
    want_s, want_c = reduce_expected(sums, counts, order, off)
    if len(off) > 1:  # the test would not see items taken in index order
        ident_s, _ = reduce_expected(sums, counts, np.arange(N), off)
        assert (ident_s.view(np.int64) != want_s.view(np.int64)).any()
    dev = cuda_device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    got_s, got_c = metrics._reduce(t(sums), t(counts), t(order), t(off), len(off) - 1, dev)
    np.testing.assert_array_equal(got_s.view(np.int64), want_s.view(np.int64))
    np.testing.assert_array_equal(got_c, want_c)
