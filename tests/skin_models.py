"""SMPL-X-shaped body models with a prescribed skinning structure, for the skinning-path tests (not collected by pytest).

``skin_model(V, tile_bones, vertex_bones, unit, seed)`` returns the tensor dict of ``synthetic.smplx_like_model``
(v_template [V,3], shapedirs [V,3,20], posedirs [486, 3V], J_regressor [55,V], lbs_weights [V,55], parents) in which
32-vertex tile t (vertices 32 t ... 32 t + 31) touches exactly ``tile_bones[t]`` distinct bones and vertex v carries exactly
``vertex_bones[v]`` of them.  Bones are drawn from all 55 joints, hands, jaw and eyes included; weights are positive,
normalised in float64 and then cast to fp32.  ``unit`` is "m" or "mm": the millimetre model is the metre model with
v_template, shapedirs and posedirs times 1000.

The weight-sum contract.  Every skinning path of rohm_body_forward folds ``transl`` into the bone transforms (A_b carries
t_b + transl), so the kernels compute  sum_b w_b (R_b v + t_b + transl) = smplx's verts + transl + (sum_b w_b - 1) transl.
That equals smplx's output only when a vertex's weights sum to 1.  fp32 weights normalised in float64 sum to 1 within
about n_b 2^-24 (n_b bones), so an error bound for vertices carries the term |sum_b w_b - 1| |transl|.

``expected_path(weights, f16)`` restates rohm_body_create's choice of skinning path from the weights alone.
"""
import numpy as np
import torch

from rohm_b200.synthetic import SMPLX_PARENTS

J = 55
TILE = 32               # vertices per column tile of the fused launch (96 columns / 3)
TILE_BONES_MAX = 16     # kSkinTileBones: bones one tile of the fused skinning epilogue can hold
VERTEX_BONES_MAX = 8    # kMaxBones: bones per vertex of the sparse skinning kernel
SKIN_FUSED, SKIN_SPARSE, SKIN_DENSE = 0, 1, 2


def tiles(V):
    return -(-int(V) // TILE)


def skin_model(V, tile_bones, vertex_bones, unit="m", seed=0):
    V = int(V)
    tile_bones = [int(b) for b in tile_bones]
    vertex_bones = [int(b) for b in vertex_bones]
    if len(tile_bones) != tiles(V) or len(vertex_bones) != V:
        raise ValueError("skin_model: one bone count per 32-vertex tile and one per vertex")
    if unit not in ("m", "mm"):
        raise ValueError("skin_model: unit is 'm' or 'mm'")
    rng = np.random.RandomState(seed)
    # bone set of tile t: a window of a seeded permutation of all 55 joints, shifted by 7 per tile, so that consecutive
    # tiles share bones (as body parts do) and every joint is used once the model has a few tiles
    perm = rng.permutation(J)
    W = np.zeros((V, J), np.float64)
    for t, nb in enumerate(tile_bones):
        lo, hi = TILE * t, min(V, TILE * (t + 1))
        if not 1 <= nb <= J:
            raise ValueError(f"skin_model: tile {t} asks for {nb} bones")
        if sum(vertex_bones[lo:hi]) < nb:
            raise ValueError(f"skin_model: the vertices of tile {t} carry fewer than its {nb} bones")
        bones = perm[(7 * t + np.arange(nb)) % J]
        cursor = 0
        for v in range(lo, hi):
            k = vertex_bones[v]
            if not 1 <= k <= nb:
                raise ValueError(f"skin_model: vertex {v} asks for {k} bones in a tile of {nb}")
            # consecutive slots of the tile's bone list: the tile's vertices cover every bone once their counts add up to nb
            W[v, bones[(cursor + np.arange(k)) % nb]] = 0.05 + rng.rand(k)
            cursor += k
    W /= W.sum(axis=1, keepdims=True)
    lbs = torch.from_numpy(W).to(torch.float32)
    # geometry as in synthetic.smplx_like_model: a random tree with 8-23 cm bones, each vertex near one of its bones
    rest = np.zeros((J, 3))
    for j in range(1, J):
        d = rng.randn(3)
        rest[j] = rest[SMPLX_PARENTS[j]] + d / np.linalg.norm(d) * (0.08 + 0.15 * rng.rand())
    owner = np.argmax(W > 0, axis=1)
    v_template = rest[owner] + 0.05 * rng.randn(V, 3)
    Jreg = np.zeros((J, V))
    for j in range(J):
        pick = rng.choice(V, size=min(V, 32), replace=False)
        w = rng.rand(pick.size)
        Jreg[j, pick] = w / w.sum()
    shapedirs = 0.01 * rng.randn(V, 3, 20)
    posedirs = 0.002 * rng.randn((J - 1) * 9, V * 3)
    s = 1000.0 if unit == "mm" else 1.0
    f = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(torch.float32)
    return {"v_template": f(s * v_template), "shapedirs": f(s * shapedirs), "posedirs": f(s * posedirs),
            "J_regressor": f(Jreg), "lbs_weights": lbs, "parents": list(SMPLX_PARENTS)}


def structure(weights):
    """(bones per 32-vertex tile, bones per vertex) of an lbs_weights tensor [V, 55]."""
    nz = torch.as_tensor(weights) != 0
    V = nz.shape[0]
    per_tile = [int(nz[TILE * t:TILE * (t + 1)].any(0).sum()) for t in range(tiles(V))]
    return per_tile, [int(c) for c in nz.sum(1)]


def expected_path(weights, f16=True):
    """rohm_body_create's rule: fused with fp16 pairs when every tile touches <= 16 bones, else sparse two-kernel when every
    vertex has <= 8 bones, else dense two-kernel."""
    per_tile, per_vertex = structure(weights)
    if f16 and max(per_tile) <= TILE_BONES_MAX:
        return SKIN_FUSED
    return SKIN_SPARSE if max(per_vertex) <= VERTEX_BONES_MAX else SKIN_DENSE


# ----- the structures the GPU tests use -----
def fused_sweep_counts(V):
    """Tile t touches t % 16 + 1 bones; each vertex carries 1 ... min(8, tile bones) bones, and the 16-bone tiles also hold
    vertices with 9 ... 16 bones (so the model is fused, but would be dense on the two-kernel path)."""
    tb = [t % 16 + 1 for t in range(tiles(V))]
    vb = []
    for v in range(V):
        t, i = divmod(v, TILE)
        cap = min(VERTEX_BONES_MAX, tb[t])
        vb.append(9 + (i // 4) % 8 if tb[t] == 16 and i % 4 == 3 else 1 + (i + t) % cap)
    return tb, vb


def fused_counts(V):
    """At most 16 bones per tile, 1 ... 8 bones per vertex: the fused path, and the sparse one without it."""
    tb = [min(16, 1 + (3 * t) % 16 + (2 if t % 5 == 0 else 0)) for t in range(tiles(V))]
    vb = [1 + (v % TILE + v // TILE) % min(VERTEX_BONES_MAX, tb[v // TILE]) for v in range(V)]
    return tb, vb


def two_kernel_counts(V, max_vertex_bones=VERTEX_BONES_MAX):
    """Vertices cycle through 1 ... max_vertex_bones bones; tile t touches 17 + (5 t) % 39 bones (17 ... 55), capped by the
    bones its vertices carry: never fused."""
    vb = [1 + v % max_vertex_bones for v in range(V)]
    tb = [min(17 + (5 * t) % 39, sum(vb[TILE * t:TILE * (t + 1)])) for t in range(tiles(V))]
    return tb, vb
