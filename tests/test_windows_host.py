"""CPU: the window rule and the float64 window oracle (oracle/windows_oracle.py) against the reference's loaders, pinned by
tests/golden/windows.npz (tools/gen_golden.py gen_windows: cano_seq_smplx -> get_repr_smplx per window, points_coord_trans
with the inverse transf_matrix)."""
import numpy as np
import pytest
import torch

from helpers import golden
from oracle import windows_oracle as wo
from rohm_b200 import windows
from rohm_b200._lib import RohmB200Error

PARAM_NAMES = ("global_orient", "transl", "betas", "body_pose")


def golden_case(g, c):
    """(clip_len, overlap, lengths, params, joints) of case c: its recordings packed in order."""
    meta = [int(v) for v in g[f"c{c}_meta"]]
    overlap, recs = meta[0], meta[1:]
    lengths = [int(n) for n in g["lengths"]]
    off = np.concatenate([[0], np.cumsum(lengths)])
    rows = np.concatenate([np.arange(off[r], off[r + 1]) for r in recs])
    params = {k: g[f"param_{k}"][rows] for k in PARAM_NAMES}
    return int(g["clip_len"]), overlap, [lengths[r] for r in recs], params, g["joints"][rows]


def amass_windows(n, clip_len):
    """dataloader_amass.py:123-129: int(N / clip_len) windows at clip_len * i when N >= clip_len."""
    return [clip_len * i for i in range(int(n / clip_len))] if n >= clip_len else []


def video_windows(n, clip_len, overlap):
    """dataloader_video.py:161-178."""
    out, seq_idx = [], 0
    while 1:
        start = seq_idx * (clip_len - overlap)
        if start + clip_len > n:
            break
        out.append(start)
        seq_idx += 1
    return out


@pytest.mark.parametrize("clip_len", [145, 17])
def test_window_rule_matches_the_reference_loops(clip_len):
    for overlap in (0, 2):
        stride = clip_len - overlap
        ns = sorted({0, 1, clip_len - 1, clip_len, clip_len + 1} |
                    {clip_len + k * stride + d for k in range(1, 6) for d in (-1, 0, 1)} |
                    {k * stride + d for k in range(1, 6) for d in (-1, 0, 1)})
        for n in ns:
            want = amass_windows(n, clip_len) if overlap == 0 else video_windows(n, clip_len, overlap)
            if overlap == 0:
                assert want == video_windows(n, clip_len, 0), n
            assert [s for _, s in windows.window_table([n], clip_len, overlap)] == want, (n, overlap)
            assert [s for _, s in wo.window_table([n], clip_len, overlap)] == want, (n, overlap)
        table = windows.window_table(ns, clip_len, overlap)
        assert table == wo.window_table(ns, clip_len, overlap)
        assert table == [(r, s) for r, n in enumerate(ns)
                         for s in (amass_windows(n, clip_len) if overlap == 0 else video_windows(n, clip_len, overlap))]


def test_oracle_matches_reference_windows():
    g = golden("windows.npz")
    for c in range(int(g["n_cases"])):
        L, overlap, lengths, params, joints = golden_case(g, c)
        table, transf, rep = wo.encode(params, joints, lengths, L, overlap)
        ref = g[f"c{c}_repr"].astype(np.float64)
        assert np.array(table).reshape(-1, 2).tolist() == g[f"c{c}_table"].tolist()
        assert np.abs(transf - g[f"c{c}_transf"]).max() < 1e-9
        # the reference's quaternion helpers run in float32 (torch .float()), its golden is stored in float32
        err = np.abs(rep - ref) / (1.0 + np.abs(ref))
        assert err[..., :290].max() < 2e-5, (c, np.unravel_index(err[..., :290].argmax(), err[..., :290].shape))
        assert np.array_equal(rep[..., 290:], ref[..., 290:])
        assert 0.1 < ref[..., 290:].mean() < 0.9  # both contact labels occur
        # canonical pose frames back to the world: the reference's points_coord_trans, and the recordings' own joints
        rt = transf[:, :3, :3]
        cano = np.stack([joints[np.arange(L) + int(np.cumsum([0] + lengths)[r]) + s] @ rt[w].T + transf[w, :3, 3]
                         for w, (r, s) in enumerate(table)])[:, :L - 2]
        world, covered = wo.to_world(cano, table, transf, lengths, L)
        back = np.concatenate([world[int(np.cumsum([0] + lengths)[r]) + s:][:L - 2][None] for r, s in table])
        assert np.abs(back - g[f"c{c}_world"]).max() < 1e-5
        assert np.abs(world[covered] - joints[covered]).max() < 1e-5
        off = np.cumsum([0] + lengths)
        for r, n in enumerate(lengths):
            want = np.zeros(n, dtype=bool)
            for rr, s in table:
                if rr == r:
                    want[s:s + L - 2] = True
            assert np.array_equal(covered[off[r]:off[r + 1]], want), (c, r)


def test_golden_exercises_the_heading_repair_and_both_thresholds():
    g = golden("windows.npz")
    rep = g["c0_repr"]
    # heading channel within 0.05 rad of +-90 deg (half of a heading near 180 deg) somewhere, never at it
    near = np.abs(np.abs(rep[..., 0]) - np.pi / 2)
    assert near.min() < 0.05 and near.min() > 5e-3
    _, _, lengths, _, joints = golden_case(g, 0)
    across = (joints[:, 1] - joints[:, 2]) + (joints[:, 17] - joints[:, 16])
    assert int((np.abs(across).sum(-1) == 0).sum()) == 3  # the frames the reference repairs
    assert np.isfinite(rep).all()


def test_refusals_without_a_device():
    p = {k: torch.zeros(145, w) for k, w in windows.PARAMS}
    for clip_len, overlap in ((145, 3), (2, 0), (161, 0), (145, -1)):
        with pytest.raises(RohmB200Error, match="clip_len"):
            windows.encode(None, p, [145], None, None, clip_len, overlap)
    with pytest.raises(RohmB200Error, match="CUDA"):
        windows.encode(None, p, [145], None, None)
