"""The SMPL-X-shaped models of tests/skin_models.py (CPU only): each has exactly the skinning structure it was asked for,
and rohm_body_create's rule sends it down the skinning path the GPU tests expect."""
import pytest
import torch

import skin_models as sm

SIZES = (55, 64, 75, 2000, 10475)


def _check_structure(m, tb, vb):
    W = m["lbs_weights"]
    assert W.dtype == torch.float32 and W.shape == (len(vb), 55)
    assert bool((W >= 0).all())
    assert sm.structure(W) == (list(tb), list(vb))
    # normalised in float64, then cast: each vertex's fp32 weights sum to 1 within its bone count x 2^-24
    s = W.double().sum(1)
    assert bool(((s - 1).abs() <= torch.tensor(vb, dtype=torch.float64) * 2.0 ** -24).all())
    V = len(vb)
    assert m["v_template"].shape == (V, 3) and m["shapedirs"].shape == (V, 3, 20)
    assert m["posedirs"].shape == (486, 3 * V) and m["J_regressor"].shape == (55, V) and len(m["parents"]) == 55


@pytest.mark.parametrize("V", SIZES)
def test_builder_makes_the_structure_it_was_asked_for(V):
    for counts, path in ((sm.fused_counts, sm.SKIN_FUSED), (sm.fused_sweep_counts, sm.SKIN_FUSED),
                         (sm.two_kernel_counts, sm.SKIN_SPARSE), (lambda n: sm.two_kernel_counts(n, 16), sm.SKIN_DENSE)):
        tb, vb = counts(V)
        m = sm.skin_model(V, tb, vb, seed=V)
        _check_structure(m, tb, vb)
        assert sm.expected_path(m["lbs_weights"]) == path
        assert sm.expected_path(m["lbs_weights"], f16=False) in (sm.SKIN_SPARSE, sm.SKIN_DENSE)
        if V >= 2000:  # every joint, hands, jaw and eyes included, drives some vertex
            assert set(m["lbs_weights"].nonzero()[:, 1].tolist()) == set(range(55))


def test_fused_sweep_structure():
    tb, vb = sm.fused_sweep_counts(10475)
    assert tb == [t % 16 + 1 for t in range(328)]
    for v, k in enumerate(vb):
        t = v // 32
        assert 1 <= k <= (16 if tb[t] == 16 else min(8, tb[t]))
    assert sorted({k for k in vb if k > 8}) == list(range(9, 17))  # the 16-bone tiles hold vertices with 9 ... 16 bones


def test_path_rule_at_its_limits():
    """16 bones in every tile is fused, one tile with 17 is sparse, and one vertex with 9 bones on top of that is dense."""
    V = 2000
    tb, vb = sm.fused_counts(V)
    tb[5], vb[5 * 32:6 * 32] = 16, [8] * 32
    m = sm.skin_model(V, tb, vb)
    assert sm.structure(m["lbs_weights"])[0][5] == 16 and sm.expected_path(m["lbs_weights"]) == sm.SKIN_FUSED
    tb[5] = 17
    m = sm.skin_model(V, tb, vb)
    assert sm.expected_path(m["lbs_weights"]) == sm.SKIN_SPARSE
    vb[5 * 32] = 9
    m = sm.skin_model(V, tb, vb)
    assert sm.expected_path(m["lbs_weights"]) == sm.SKIN_DENSE
    assert sm.expected_path(sm.skin_model(V, *sm.fused_counts(V))["lbs_weights"], f16=False) == sm.SKIN_SPARSE


def test_millimetre_model_is_the_metre_model_scaled():
    tb, vb = sm.fused_counts(75)
    m, mm = sm.skin_model(75, tb, vb, "m", 3), sm.skin_model(75, tb, vb, "mm", 3)
    for k in ("v_template", "shapedirs", "posedirs"):
        assert torch.allclose(mm[k].double(), 1000 * m[k].double(), rtol=2.0 ** -23, atol=0)
    assert torch.equal(mm["lbs_weights"], m["lbs_weights"]) and torch.equal(mm["J_regressor"], m["J_regressor"])


def test_builder_refuses_a_structure_it_cannot_make():
    with pytest.raises(ValueError):
        sm.skin_model(32, [17], [1] * 16 + [0] * 16)  # a vertex without bones
    with pytest.raises(ValueError):
        sm.skin_model(32, [40], [1] * 32)               # 32 one-bone vertices cannot cover 40 bones
    with pytest.raises(ValueError):
        sm.skin_model(32, [4], [5] + [1] * 31)          # a vertex with more bones than its tile
