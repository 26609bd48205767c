"""Every skinning path of rohm_body_forward against smplx's forward in float64, for every frame.

rohm_body_create picks one of three paths from the model's weights (rohm_body_skin_path): fused (blend GEMM with the
skinning epilogue, fp16 pairs, <= 16 bones per 32-vertex tile), sparse two-kernel (blend GEMM -> v_posed chunks ->
skin_kernel, <= 8 bones per vertex) and dense two-kernel (skin_dense_kernel).  The models come from tests/skin_models.py,
which builds SMPL-X-shaped models with a prescribed number of bones per tile and per vertex.  The reference is
oracle.kinematics_oracle.smplx_forward in float64 on the device, run in chunks of frames.

Error bounds.  u = 2^-24.  Every term is an operation count x u (or a pair precision) x the float64 magnitude of what the
kernel summed, so the bounds follow the model's units and the size of transl, betas and the angles:
  FK.  A local rotation from fp32 Rodrigues has entries within e_rot = (8 + 4 theta) u (theta = the frame's largest angle:
    fp32 rounds the angle itself).  Composing down the tree adds one rotation error and one 3-term product per level:
    dR_j = dR_parent + 3 (e_rot + 2 u), so the bound grows with the depth of joint j's chain.  Rest joints come from an
    fp32 regression: dJ = 64 u sum_v |Jreg| (|v_template| + sum_l |shapedirs| |beta_l|).  World translations
    dWt_j = dWt_parent + dR_parent |J_j - J_parent|_1 + 3 (dJ_j + dJ_parent) + 4 u L_j, with L_j the sum of |J_k - J_parent|_1
    along the chain (which bounds |Wt_j|).  Joints: dWt_j + u (L_j + |transl|).  The skinning translation
    t_b = Wt_b - R_b J_b + transl: dt_b = dWt_b + dR_b |J_b|_1 + 3 dJ_b + 4 u (L_b + |J_b|_1 + |transl|).
  Blend (v_posed = feat . blend, K = 200).  As in test_gpu_gemm.py: c 2^-20 sum_k |feat_k| |blend_k| with c = 2 for fp16
    and TF32 pairs and c = 2^10 for single-pass TF32 (both operands rounded to 11 bits, 2^-11 each), plus the pairs'
    absolute floors 2^-25 sum_k |blend_k| (feat lo halves) and 2^-25 / s sum_k |feat_k| (blend lo halves; s is the blend's
    single power-of-two fp16 scale, the smallest of posedirs', shapedirs' and v_template's), plus the pose features' own
    error (e_rot + u) sum_{k < 189} |blend_k|.
  Skinning.  (n_v + 5) u sum_b w_b (|R_b| |v_posed| + |t_b|) for a vertex with n_v bones (three FMAs per bone transform,
    one per weighted bone; the two-kernel paths sum the weighted transforms first and apply them after, the same count),
    plus the propagated errors sum_b w_b (dR_b |v_posed|_1 + dt_b) and (sum_b w_b) |dv_posed|_1.
  Weight sum.  Every path folds transl into the bone transforms, so it computes smplx's vertices plus
    (sum_b w_b - 1) transl (tests/skin_models.py, DESIGN.md section 4.3): the bound carries |sum_b w_b - 1| |transl|.
Each check prints the largest |error| / bound it saw.
"""
import gc
import math

import pytest
import torch

import skin_models as sm
from oracle import kinematics_oracle as ko
from rohm_b200 import _lib, glue, synthetic
from rohm_b200.body_model import BodyKernels, BodyModel

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
CHUNK = 256  # frames per float64 reference chunk: its [N, V, 4, 4] transforms are 343 MB at V = 10475
PARENTS = synthetic.SMPLX_PARENTS
ANGLES = (0.0, 1e-8, 1e-4, math.pi - 1e-4, math.pi, math.pi + 1e-4, 2 * math.pi, 3 * math.pi, 20.0)
SWITCHES = ("ROHM_B200_FUSED_LBS", "ROHM_B200_DENSE_SKIN", "ROHM_B200_LBS_CHUNK", "ROHM_B200_LBS_OVERLAP",
            "ROHM_B200_LBS_TMA_STORE")

_models = {}


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """The float64 model copies and the gigabyte-sized outputs go back to the driver when the module ends, so that the modules
    after it meet the caching allocator as they would without it."""
    yield
    _models.clear()
    _dev_models.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _model(kind, V=10475, unit="m"):
    """The CPU fp32 tensor dict of a skin_models structure, built once per (kind, V, unit)."""
    key = (kind, V, unit)
    if key not in _models:
        counts = {"sweep": sm.fused_sweep_counts, "fused": sm.fused_counts, "sparse": sm.two_kernel_counts,
                  "dense": lambda n: sm.two_kernel_counts(n, 16)}[kind]
        t = sm.skin_model(V, *counts(V), unit=unit, seed=V + len(kind))
        _models[key] = t
    return _models[key]


def _handle(monkeypatch, t, dev, cap, with_vertices=True, precision=_lib.PRECISION_F16X2, **env):
    """A fresh handle created under the given switches (rohm_body_create reads them with getenv)."""
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))
    return BodyKernels(BodyModel(t), dev, cap, with_vertices, precision)


def _params(N, seed, dev, angle=0.5, betas=1.0, transl=1.0):
    g = torch.Generator().manual_seed(seed)
    go, bp = angle * torch.randn(N, 3, generator=g), angle * torch.randn(N, 63, generator=g)
    be, tr = betas * (2 * torch.rand(N, 10, generator=g) - 1), transl * (2 * torch.rand(N, 3, generator=g) - 1)
    return [x.to(dev) for x in (go, bp, be, tr)]


def _edge_angles(N, seed, dev):
    """Every body joint of frame f gets the norm ANGLES[(f + j) % 9] on a random axis."""
    g = torch.Generator().manual_seed(seed)
    axis = torch.nn.functional.normalize(torch.randn(N, 22, 3, generator=g, dtype=torch.float64), dim=-1)
    norms = torch.tensor(ANGLES, dtype=torch.float64)[(torch.arange(N)[:, None] + torch.arange(22)[None]) % len(ANGLES)]
    aa = (axis * norms[..., None]).float()
    return aa[:, 0].contiguous().to(dev), aa[:, 1:].reshape(N, 63).to(dev)


# ---------------------------------------------------------------------------------------------------------------------
# float64 reference and bounds
# ---------------------------------------------------------------------------------------------------------------------
_dev_models = {}


def _model64(t, dev):
    """float64 device copy of a model with the sums the bounds use (the entry keeps t alive, so its id stays unique)."""
    key = id(t)
    if key not in _dev_models:
        _dev_models.clear()  # one model's float64 copy at a time (posedirs alone is 120 MB at V = 10475)
        m = {k: (v.to(device=dev, dtype=torch.float64) if torch.is_tensor(v) else v) for k, v in t.items()}
        V = m["v_template"].shape[0]
        blend = torch.cat([m["posedirs"][:189], m["shapedirs"][:, :, :10].permute(2, 0, 1).reshape(10, 3 * V),
                           m["v_template"].reshape(1, 3 * V)])                                   # [200, 3V]
        wmax = max(float(t["posedirs"][:189].abs().max()), float(t["shapedirs"].abs().max()),
                   float(t["v_template"].abs().max()))
        W = m["lbs_weights"]
        m.update(blend_abs=blend.abs(), blend_col=blend.abs().sum(0), pose_col=blend[:189].abs().sum(0),
                 scale=2.0 ** (14 - math.frexp(wmax)[1]), nb=(W != 0).sum(1).to(torch.float64), wsum=W.sum(1),
                 src=t)
        _dev_models[key] = m
    return _dev_models[key]


def _reference(m, go, bp, be, tr, passes):
    """float64 joints [n,55,3], vertices [n,V,3] and their bounds for one chunk of frames."""
    n = go.shape[0]
    go, bp, be, tr = (x.to(torch.float64) for x in (go, bp, be, tr))
    j64, v64 = ko.smplx_forward(m, go, bp, be, tr, return_verts=True)
    dev = go.device
    full = torch.cat([go.view(n, 1, 3), bp.view(n, 21, 3), torch.zeros(n, 33, 3, dtype=torch.float64, device=dev)], 1)
    e_rot = U * (8.0 + 4.0 * full.norm(dim=-1).amax(1))                                            # [n]
    sc = torch.cat([be, torch.zeros_like(be)], -1)
    v_shaped = m["v_template"] + torch.einsum('bl,mkl->bmk', sc, m["shapedirs"])
    Jr = torch.einsum('bik,ji->bjk', v_shaped, m["J_regressor"])
    mag = m["v_template"].abs() + torch.einsum('bl,mkl->bmk', sc.abs(), m["shapedirs"].abs())
    dJ = 64 * U * torch.einsum('bik,ji->bjk', mag, m["J_regressor"].abs()).amax(-1)              # [n,55]
    R = ko.batch_rodrigues(full.reshape(-1, 3)).view(n, 55, 3, 3)
    _, A = ko.batch_rigid_transform(R, Jr, PARENTS)
    rel = Jr.clone()
    rel[:, 1:] -= Jr[:, PARENTS[1:]]
    relm, Jm = rel.abs().sum(-1), Jr.abs().sum(-1)
    trm = tr.abs().amax(-1)
    L, dR, dWt = torch.zeros_like(relm), torch.zeros_like(relm), torch.zeros_like(relm)
    for j in range(55):
        p = PARENTS[j]
        if p < 0:
            L[:, j], dR[:, j], dWt[:, j] = relm[:, j], 3 * (e_rot + 2 * U), dJ[:, j]
        else:
            L[:, j] = L[:, p] + relm[:, j]
            dR[:, j] = dR[:, p] + 3 * (e_rot + 2 * U)
            dWt[:, j] = dWt[:, p] + dR[:, p] * relm[:, j] + 3 * (dJ[:, j] + dJ[:, p]) + 4 * U * L[:, j]
    bj = dWt[..., None] + U * (L[..., None] + tr.abs()[:, None, :])
    dt = dWt + dR * Jm + 3 * dJ + 4 * U * (L + Jm + trm[:, None])
    # blend
    feat = torch.cat([(R[:, 1:22] - torch.eye(3, dtype=torch.float64, device=dev)).reshape(n, 189), be,
                      torch.ones(n, 1, dtype=torch.float64, device=dev)], 1)
    c = 2.0 if passes == 3 else 2.0 ** 10
    dvp = (c * 2.0 ** -20 * (feat.abs() @ m["blend_abs"]) + 2.0 ** -25 * m["blend_col"]
           + 2.0 ** -25 / m["scale"] * feat.abs().sum(1, keepdim=True) + (e_rot + U)[:, None] * m["pose_col"])
    V = m["v_template"].shape[0]
    dvp = dvp.view(n, V, 3).sum(-1)                                                              # |dv_posed|_1
    vp = v_shaped + (feat[:, :189] @ m["posedirs"][:189]).view(n, V, 3)
    # skinning
    W = m["lbs_weights"]
    tb = A[:, :, :3, 3] + tr[:, None, :]                                                       # transl folded in
    absA = torch.cat([A[:, :, :3, :3].abs().reshape(n, 55, 9), tb.abs()], -1)                  # [n,55,12]
    T = torch.einsum('vb,nbe->nve', W, absA)
    S = (T[..., :9].view(n, V, 3, 3) @ vp.abs()[..., None])[..., 0] + T[..., 9:]
    bv = ((m["nb"] + 5)[None, :, None] * U * S
          + ((W @ dR.T).T[..., None] * vp.abs().sum(-1, keepdim=True) + (W @ dt.T).T[..., None])
          + (m["wsum"][None, :, None] * dvp[..., None])
          + (m["wsum"] - 1).abs()[None, :, None] * tr.abs()[:, None, :])
    return j64, v64, bj, bv


def _check(t, dev, inputs, joints, verts, what, passes=3, frames=None):
    """Every frame's joints and vertices within the bound; frames: the frame indices to check (default all)."""
    m = _model64(t, dev)
    go, bp, be, tr = inputs
    N = go.shape[0]
    idx = torch.arange(N, device=dev) if frames is None else torch.as_tensor(frames, device=dev)
    rj = rv = 0.0
    for s in range(0, idx.numel(), CHUNK):
        f = idx[s:s + CHUNK]
        j64, v64, bj, bv = _reference(m, go[f], bp[f], be[f], tr[f], passes)
        if joints is not None:
            nj = joints.shape[1]
            gj = joints[f].double()
            assert bool(torch.isfinite(gj).all()), what
            rj = max(rj, float(((gj - j64[:, :nj]).abs() / bj[:, :nj]).max()) if nj else 0.0)
        if verts is not None:
            gv = verts[f].double()
            assert bool(torch.isfinite(gv).all()), what
            rv = max(rv, float(((gv - v64).abs() / bv).max()))
    print(f"{what}: max |err| / bound: joints {rj:.3f}, vertices {rv:.3f}")
    assert rj <= 1.0 and rv <= 1.0, (what, rj, rv)
    return rj, rv


def _bits(x):
    return x.contiguous().view(torch.int32)


# ---------------------------------------------------------------------------------------------------------------------
def test_device_reference_matches_the_cpu_reference(cuda_device):
    t = _model("sweep")
    go, bp, be, tr = _params(3, 1, "cpu", angle=1.0, betas=3.0, transl=10.0)
    jc, vc = ko.smplx_forward(t, go, bp, be, tr, return_verts=True, dtype=torch.float64)
    jd, vd = ko.smplx_forward(t, *(x.to(cuda_device) for x in (go, bp, be, tr)), return_verts=True, dtype=torch.float64)
    assert jd.device == vd.device == cuda_device
    assert float((jd.cpu() - jc).abs().max()) <= 1e-12 and float((vd.cpu() - vc).abs().max()) <= 1e-12


def test_each_model_takes_its_skinning_path(cuda_device, monkeypatch):
    """16 bones in every tile -> fused; one tile with 17 -> sparse; one vertex with 9 on top -> dense; TF32 handles are
    never fused; a handle without vertices has no path.  Every model's vertices are then within the bound."""
    V, N = 2000, 33
    tb, vb = sm.fused_counts(V)
    tb[5], vb[5 * 32:6 * 32] = 16, [8] * 32
    fused = sm.skin_model(V, tb, vb, seed=11)
    tb[5] = 17
    sparse = sm.skin_model(V, tb, vb, seed=12)
    vb[5 * 32] = 9
    dense = sm.skin_model(V, tb, vb, seed=13)
    inputs = _params(N, 3, cuda_device)
    for t, path in ((fused, _lib.SKIN_FUSED), (sparse, _lib.SKIN_SPARSE), (dense, _lib.SKIN_DENSE)):
        assert sm.expected_path(t["lbs_weights"]) == path
        for prec in (_lib.PRECISION_F16X2, _lib.PRECISION_TF32X3, _lib.PRECISION_TF32):
            k = _handle(monkeypatch, t, cuda_device, N, precision=prec)
            want = sm.expected_path(t["lbs_weights"], f16=prec == _lib.PRECISION_F16X2)
            assert k.lib.rohm_body_skin_path(k.handle) == k.skin_path == want, (path, prec)
            assert prec == _lib.PRECISION_F16X2 or want != _lib.SKIN_FUSED
            j, v = k.forward(*inputs, True)
            _check(t, cuda_device, inputs, j, v, f"path {want} precision {prec}", passes=1 if prec == _lib.PRECISION_TF32 else 3)
            del k
    k = _handle(monkeypatch, fused, cuda_device, N, with_vertices=False)
    assert k.lib.rohm_body_skin_path(k.handle) == k.skin_path == -1


def test_fused_bone_sweep(cuda_device, monkeypatch):
    """Tile t touches t % 16 + 1 bones (1 ... 4 kept in registers, 5 ... 16 read from L2 one bone ahead), vertices carry
    1 ... 16 bones; capacity 4577 frames (not a multiple of 128), the pitched TMA store and the dense store."""
    t = _model("sweep")
    cap = 4577
    out = {}
    for store in ("1", "0"):
        k = _handle(monkeypatch, t, cuda_device, cap, ROHM_B200_LBS_TMA_STORE=store)
        assert k.skin_path == _lib.SKIN_FUSED and bool(k.vertex_pitch) == (store == "1")
        for N in (1, 127, 129, 300, 4577):
            inputs = _params(N, 100 + N, cuda_device)
            j, v = k.forward(*inputs, True)
            if store == "1":
                _check(t, cuda_device, inputs, j, v, f"fused sweep N={N}")
                out[N] = (j, v)
            else:
                assert torch.equal(_bits(out[N][0]), _bits(j)) and torch.equal(_bits(out[N][1]), _bits(v)), N
                del out[N]
        del k


@pytest.mark.parametrize("kind", ["sparse", "dense"])
def test_two_kernel_chunks(cuda_device, monkeypatch, kind):
    """N = 1, 129, 4608 (one default chunk) and 4609 (two); chunks of 128 and 384 frames (odd and even chunk counts) and
    the serial single-stream pipeline give the default's bits, which are within the bound.  On the sparse model the dense
    skinning kernel gives the same bits as skin_kernel."""
    t = _model(kind)
    path = _lib.SKIN_SPARSE if kind == "sparse" else _lib.SKIN_DENSE
    sizes = (1, 129, 4608, 4609)
    cap = max(sizes)
    k = _handle(monkeypatch, t, cuda_device, cap)
    assert k.skin_path == path
    base = {}
    for N in sizes:
        inputs = _params(N, 200 + N, cuda_device)
        base[N] = k.forward(*inputs, True)
        _check(t, cuda_device, inputs, *base[N], f"{kind} N={N}")
    del k
    variants = [{"ROHM_B200_LBS_CHUNK": 128}, {"ROHM_B200_LBS_CHUNK": 384}, {"ROHM_B200_LBS_OVERLAP": 0},
                {"ROHM_B200_LBS_CHUNK": 128, "ROHM_B200_LBS_OVERLAP": 0}]
    if kind == "sparse":
        variants.append({"ROHM_B200_DENSE_SKIN": 1})
    for env in variants:
        k = _handle(monkeypatch, t, cuda_device, cap, **env)
        assert k.skin_path == (_lib.SKIN_DENSE if "ROHM_B200_DENSE_SKIN" in env else path)
        for N in sizes:
            j, v = k.forward(*_params(N, 200 + N, cuda_device), True)
            assert torch.equal(_bits(j), _bits(base[N][0])) and torch.equal(_bits(v), _bits(base[N][1])), (env, N)
        del k


@pytest.mark.parametrize("V", [55, 64, 75, 2000, 10475])
def test_vertex_counts(cuda_device, monkeypatch, V):
    """3V mod 96 in {69, 0, 33, 48}, column tiles past the last vertex, last tiles of 23, 32, 11 and 16 vertices, and
    3V mod 4 != 0 for the pitched store; on the fused path (both stores) and the two-kernel path."""
    for kind, path in (("fused", _lib.SKIN_FUSED), ("sparse", _lib.SKIN_SPARSE)):
        t = _model(kind, V)
        for store in ("1", "0"):
            if store == "0" and path != _lib.SKIN_FUSED:
                continue
            k = _handle(monkeypatch, t, cuda_device, 129, ROHM_B200_LBS_TMA_STORE=store)
            assert k.skin_path == path
            for N in (1, 129):
                inputs = _params(N, V + N, cuda_device)
                j, v = k.forward(*inputs, True)
                assert v.shape == (N, V, 3)
                _check(t, cuda_device, inputs, j, v, f"{kind} V={V} store {store} N={N}")
            del k


@pytest.mark.parametrize("kind", ["sweep", "sparse", "dense"])
def test_edge_angles(cuda_device, monkeypatch, kind):
    """Axis-angle norms 0, 1e-8, 1e-4, pi - 1e-4, pi, pi + 1e-4, 2 pi, 3 pi and 20 on random axes, on every body joint."""
    t = _model(kind)
    N = 9 * 16
    k = _handle(monkeypatch, t, cuda_device, N)
    go, bp = _edge_angles(N, 5, cuda_device)
    _, _, be, tr = _params(N, 6, cuda_device)
    j, v = k.forward(go, bp, be, tr, True)
    _check(t, cuda_device, (go, bp, be, tr), j, v, f"{kind} edge angles")


@pytest.mark.parametrize("unit", ["m", "mm"])
@pytest.mark.parametrize("kind", ["fused", "sparse"])
def test_large_betas_and_transl(cuda_device, monkeypatch, kind, unit):
    """Betas up to +-5 and transl up to +-1e3, in a metre and a millimetre model (whose v_template sets the blend's single
    fp16 scale)."""
    t = _model(kind, 2000, unit)
    N = 129
    k = _handle(monkeypatch, t, cuda_device, N)
    inputs = _params(N, 7, cuda_device, angle=1.0, betas=5.0, transl=1e3)
    j, v = k.forward(*inputs, True)
    _check(t, cuda_device, inputs, j, v, f"{kind} {unit} betas 5 transl 1e3")


@pytest.mark.parametrize("kind", ["fused", "sparse"])
def test_num_joints_and_joints_only_handle(cuda_device, monkeypatch, kind):
    """num_joints 0, 1, 22, 24, 55 return the first joints of the 55 with the same bits, the vertices do not change, and a
    handle without vertices computes the same joints."""
    t = _model(kind, 2000)
    N = 129
    inputs = _params(N, 8, cuda_device)
    k = _handle(monkeypatch, t, cuda_device, N)
    j55, v55 = k.forward(*inputs, True)
    _check(t, cuda_device, inputs, j55, v55, f"{kind} 55 joints")
    kj = _handle(monkeypatch, t, cuda_device, N, with_vertices=False)
    assert kj.skin_path == -1
    for nj in (0, 1, 22, 24, 55):
        j, v = k.forward(*inputs, True, num_joints=nj)
        assert j.shape == (N, nj, 3)
        assert torch.equal(_bits(j), _bits(j55[:, :nj])) and torch.equal(_bits(v), _bits(v55)), nj
        if nj:
            jo, vo = kj.forward(*inputs, False, num_joints=nj)
            assert vo is None and torch.equal(_bits(jo), _bits(j55[:, :nj])), nj


@pytest.mark.parametrize("kind", ["fused", "sparse", "dense"])
def test_non_finite_inputs_stay_in_their_frame(cuda_device, monkeypatch, kind):
    """NaN, +Inf or -Inf in one frame's global_orient, body_pose, betas or transl: every other frame's joints and vertices
    keep the clean call's bits.  Frames 0, 127, 128 and the last; on the two-kernel paths (128-frame chunks) also 256, the
    first frame of the third chunk."""
    t = _model(kind, 2000)
    N = 300
    env = {} if kind == "fused" else {"ROHM_B200_LBS_CHUNK": 128}
    k = _handle(monkeypatch, t, cuda_device, N, **env)
    clean = _params(N, 9, cuda_device)
    j0, v0 = k.forward(*clean, True)
    j0, v0 = j0.clone(), v0.clone()
    frames = (0, 127, 128, N - 1) + (() if kind == "fused" else (256,))
    for f in frames:
        keep = torch.ones(N, dtype=torch.bool, device=cuda_device)
        keep[f] = False
        for p in range(4):
            for bad in (float("nan"), float("inf"), float("-inf")):
                x = [c.clone() for c in clean]
                x[p][f, p % x[p].shape[1]] = bad
                j, v = k.forward(*x, True)
                assert torch.equal(_bits(j[keep]), _bits(j0[keep])) and torch.equal(_bits(v[keep]), _bits(v0[keep])), (f, p, bad)


@pytest.mark.parametrize("precision", [_lib.PRECISION_TF32X3, _lib.PRECISION_TF32])
def test_tf32_handles(cuda_device, monkeypatch, precision):
    """TF32 pairs meet the pair bound, single-pass TF32 the bound of a 2^-11-relative operand rounding; neither is fused."""
    t = _model("fused")
    N = 300
    k = _handle(monkeypatch, t, cuda_device, N, precision=precision)
    assert k.skin_path == _lib.SKIN_SPARSE
    inputs = _params(N, 10, cuda_device)
    j, v = k.forward(*inputs, True)
    _check(t, cuda_device, inputs, j, v, f"precision {precision}", passes=3 if precision == _lib.PRECISION_TF32X3 else 1)


def test_packed_recovery_across_chunks(cuda_device, monkeypatch):
    """from_repr with lengths on the two-kernel path in 128-frame chunks: 423 packed frames (four chunks) are the padded
    call's frames, bit for bit."""
    t = _model("sparse", 2000)
    lengths, T = (145, 100, 145, 33), 145
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    x = synthetic.plausible_motion(len(lengths), T, 21, ds).to(cuda_device)
    mean, std = glue.stats_on(ds, cuda_device)
    k = _handle(monkeypatch, t, cuda_device, len(lengths) * T, ROHM_B200_LBS_CHUNK=128)
    assert k.skin_path == _lib.SKIN_SPARSE
    jp, vp = k.from_repr(x, mean, std, want_vertices=True)
    L = glue.device_lengths(lengths, cuda_device)
    j, v = k.from_repr(x, mean, std, want_vertices=True, lengths=L)
    assert v.shape == (sum(lengths), 2000, 3) and sum(lengths) > 3 * 128
    for b, (jb, vb) in enumerate(zip(glue.split_clips(j, L), glue.split_clips(v, L))):
        n = lengths[b]
        assert torch.equal(_bits(jb), _bits(jp[b, :n])) and torch.equal(_bits(vb), _bits(vp[b, :n])), b
