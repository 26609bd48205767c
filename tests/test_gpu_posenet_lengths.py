"""PoseNet on batches of clips with different lengths (batch['lengths']): every clip's frames equal the clip run alone, bit
for bit, padded frames are zero and their inputs never matter; the packed attention launches against float64 through the
kernel probe; the length-masked skating guidance against the float64 oracle; and the refusals."""
import argparse
import math

import pytest
import torch

import kernel_probe as kp
import packed_attention_probe as pap
from oracle import masked_skating_oracle
from rohm_b200 import _lib, diffusion, synthetic
from rohm_b200._lib import RohmB200Error
from rohm_b200.body_model import kernels_for
from rohm_b200.posenet import PoseNet
from test_gpu_attention import C_OUT, SENTINEL, _split_ok

pytestmark = pytest.mark.gpu

D, H, DH = 512, 4, 128


def _model(dev, ds=None, num_heads=H):
    ds = ds if ds is not None else synthetic.make_dataset('pose')
    m = PoseNet(dataset=ds, body_feat_dim=294, latent_dim=D, ff_size=1024, num_layers=8, num_heads=num_heads, device=dev,
                traj_feat_dim=22)
    m.load_state_dict({k: v.cpu() for k, v in synthetic.synth_state_dict(m, 1).items()})
    return m.to(dev).eval()


@pytest.fixture(scope="module")
def posenet(cuda_device):
    return _model(cuda_device)


def _inputs(B, T, seed, dev):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 294, 1, T, generator=g).to(dev)
    cond = synthetic.posenet_batch(B, T, seed)['cond'].to(dev)
    ts = torch.randint(0, 1000, (B,), generator=g).to(dev)
    return x, cond, ts


def _bits(t):
    return t.contiguous().view(torch.int32)


def _poison(t, lengths):
    """A copy with every padded frame filled with NaN, +Inf, -Inf and 1e30 in turn."""
    t = t.clone()
    vals = torch.tensor([float("nan"), float("inf"), float("-inf"), 1e30], device=t.device)
    T = t.shape[-1]
    for b, L in enumerate(lengths):
        if L < T:
            t[b, ..., L:] = vals[torch.arange(L, T, device=t.device) % 4]
    return t


def test_ragged_forward_equals_each_clip_alone(posenet, cuda_device):
    """T = 1000 with clips on both sides of the 160-token switch (159 / 160 frames = 160 / 161 tokens) and of the 64-key
    blocks: real frames bit-identical to the clip alone, padded frames exactly zero, and the same bits when the padded
    frames of x_t and cond hold NaN, +-Inf and 1e30."""
    m = posenet
    lengths = [1, 7, 143, 159, 160, 1000]
    B, T = len(lengths), 1000
    x, cond, ts = _inputs(B, T, 11, cuda_device)
    L = torch.tensor(lengths, device=cuda_device)
    out = m({'x_t': x, 'cond': cond, 'lengths': L}, ts)
    for b, n in enumerate(lengths):
        alone = m({'x_t': x[b:b + 1, ..., :n].contiguous(), 'cond': cond[b:b + 1, ..., :n].contiguous()}, ts[b:b + 1])
        assert torch.equal(_bits(out[b:b + 1, ..., :n]), _bits(alone)), f"clip {b} ({n} frames) differs from the clip alone"
        assert bool((out[b, ..., n:] == 0).all()), f"clip {b}: padded frames are not zero"
    out2 = m({'x_t': _poison(x, lengths), 'cond': _poison(cond, lengths), 'lengths': L}, ts)
    assert torch.equal(_bits(out2), _bits(out)), "values in padded frames reached a real frame"


@pytest.mark.parametrize("B,T", [(3, 145), (2, 300)])
def test_uniform_lengths_equal_no_lengths(posenet, cuda_device, B, T):
    """lengths = T for every clip gives the bits of the batch without the key; a forward without the key after one with
    it gives them too (the engine returns to uniform clips)."""
    m = posenet
    x, cond, ts = _inputs(B, T, 20 + T, cuda_device)
    ref = m({'x_t': x, 'cond': cond}, ts).clone()
    got = m({'x_t': x, 'cond': cond, 'lengths': torch.full((B,), T, dtype=torch.int32, device=cuda_device)}, ts).clone()
    assert torch.equal(_bits(got), _bits(ref))
    again = m({'x_t': x, 'cond': cond}, ts)
    assert torch.equal(_bits(again), _bits(ref))


class _SlicedTape:
    """Seeded noise for a padded [B, C, 1, T] batch, draw by draw; with clip=(b, n) every draw is the slice
    [b:b+1, ..., :n] of the same padded draw, as a clip run alone on its slice of the batch's noise sees it."""

    def __init__(self, seed, full_shape, device, clip=None):
        self.seed, self.full, self.device, self.clip, self.k = seed, tuple(full_shape), device, clip, 0

    def _draw(self, shape):
        z = torch.randn(self.full, generator=torch.Generator().manual_seed(1000 * self.seed + self.k))
        self.k += 1
        if self.clip is not None:
            b, n = self.clip
            z = z[b:b + 1, ..., :n]
        assert tuple(z.shape) == tuple(shape), (z.shape, shape)
        return z.contiguous().to(self.device)

    def randn(self, *shape, device=None, **kw):
        return self._draw(shape)

    def randn_like(self, x):
        return self._draw(x.shape)


def _diff(dev):
    args = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    return diffusion.create_gaussian_diffusion(args, diffusion, diffusion.SpacedDiffusionPoseNet, 1000, '20', dev)


def test_ragged_sampling_equals_each_clip_alone(posenet, cuda_device):
    """A 20-step respaced p_sample_loop over a ragged batch, noise injected through the diffusion object's hooks: every
    clip equals its loop run alone on its slice of the same noise, bit for bit; the final sample's padded frames are
    zero."""
    m = posenet
    lengths = [40, 161, 300]
    B, T = len(lengths), 300
    shape = (B, 294, 1, T)
    _, cond, _ = _inputs(B, T, 31, cuda_device)
    d = _diff(cuda_device)
    tape = _SlicedTape(5, shape, cuda_device)
    d._randn, d._randn_like = tape.randn, tape.randn_like
    batch = {'cond': cond, 'lengths': torch.tensor(lengths, device=cuda_device)}
    out = d.p_sample_loop(m, batch, list(shape), clip_denoised=False)
    for b, n in enumerate(lengths):
        d1 = _diff(cuda_device)
        t1 = _SlicedTape(5, shape, cuda_device, clip=(b, n))
        d1._randn, d1._randn_like = t1.randn, t1.randn_like
        alone = d1.p_sample_loop(m, {'cond': cond[b:b + 1, ..., :n].contiguous()}, [1, 294, 1, n], clip_denoised=False)
        assert torch.equal(_bits(out[b:b + 1, ..., :n]), _bits(alone)), f"clip {b} ({n} frames)"
        assert bool((out[b, ..., n:] == 0).all()), f"clip {b}: padded frames of the final sample are not zero"


# ---------------------------------------------------------------------------------------------------------------------
# skating guidance with lengths
# ---------------------------------------------------------------------------------------------------------------------
def _motion(B, T, seed):
    ds = synthetic.make_dataset('pose', seed=3, realistic_std=True)
    return ds, synthetic.plausible_motion(B, T, seed, ds)


def _guidance_setup(cuda_device, B, T, seed):
    ds, x = _motion(B, T, seed)
    m = _model(cuda_device, ds)
    mean, std = torch.from_numpy(ds.Mean).to(cuda_device), torch.from_numpy(ds.Std).to(cuda_device)
    k = kernels_for(m.smplx_model, cuda_device, B * T, with_vertices=False)
    return ds, x, m, mean, std, k


def test_guidance_with_full_lengths_equals_the_existing_entry_point(cuda_device):
    B, T = 3, 50
    _, x, m, mean, std, k = _guidance_setup(cuda_device, B, T, 2)
    xg = x.to(cuda_device)
    ref = k.skating_guidance(xg, mean, std)
    got = k.skating_guidance(xg, mean, std, lengths=torch.full((B,), T, dtype=torch.int32, device=cuda_device))
    assert float(ref.abs().max()) > 0
    assert torch.equal(_bits(got), _bits(ref))
    hook = m.guide_skating_with_smpl({'lengths': torch.full((B,), T, device=cuda_device)}, {'pred_xstart': xg}, None,
                                     compute_grad='x_0')
    assert torch.equal(_bits(hook), _bits(ref))


def test_guidance_of_one_padded_clip_equals_the_clip_alone(cuda_device):
    """B = 1, 37 of 60 frames real, the padded frames NaN / Inf: equal to the clip alone within 1e-6 relative (the sums
    may be reduced in another order), zero past the clip."""
    n, T = 37, 60
    _, x, m, mean, std, k = _guidance_setup(cuda_device, 1, T, 7)
    xg = _poison(x.to(cuda_device), [n])
    alone = k.skating_guidance(xg[..., :n].contiguous(), mean, std)
    got = k.skating_guidance(xg, mean, std, lengths=torch.tensor([n], dtype=torch.int32, device=cuda_device))
    scale = float(alone.abs().max())
    assert scale > 0
    assert float((got[..., :n] - alone).abs().max()) <= 1e-6 * scale
    assert bool((got[..., n:] == 0).all())


def test_ragged_guidance_matches_the_masked_float64_oracle(cuda_device):
    """3 clips of 50, 23 and 9 real frames against oracle.masked_skating_oracle.guide_skating_lengths (float64 autograd), within
    the bound test_gpu_body.py uses for the unmasked gradient."""
    lengths = [50, 23, 9]
    B, T = 3, 50
    ds, x, m, mean, std, k = _guidance_setup(cuda_device, B, T, 2)
    xg = x.to(cuda_device)
    got = m.guide_skating_with_smpl({'x_t': xg, 'lengths': torch.tensor(lengths, device=cuda_device)},
                                    {'pred_xstart': xg}, None, compute_grad='x_0').cpu()
    ref = masked_skating_oracle.guide_skating_lengths(x.double(), torch.from_numpy(ds.Mean).double(), torch.from_numpy(ds.Std).double(),
                                   synthetic.smplx_like_model(0), lengths)
    assert ref.dim() > 0, "nothing skates in this input"
    scale = float(ref.abs().max())
    assert float((got.double() - ref).abs().max()) < 2e-4 * scale
    for b, n in enumerate(lengths):
        assert bool((got[b, ..., n:] == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# packed attention through the kernel probe
# ---------------------------------------------------------------------------------------------------------------------
SHORT = [1, 63, 64, 65, 145, 160]       # tokens: the 160-key kernel
LONG = [161, 200, 257, 1000]            # tokens: the streaming kernel
POISONED_CLIP = 2                       # a clip of NaN: nothing of it may reach another clip
UNLISTED_CLIP = 5                       # in the packed buffer but in no launch: its rows stay untouched


def _packed(dev, tokens, seed):
    g = torch.Generator().manual_seed(seed)
    off = [0]
    for s in tokens:
        off.append(off[-1] + s)
    rows = off[-1] + 37
    qkv = torch.full((rows, 3 * D), float("nan"))
    qkv[:off[-1]] = torch.randn(off[-1], 3 * D, generator=g)
    qkv[off[POISONED_CLIP]:off[POISONED_CLIP + 1]] = float("nan")
    hi, lo = kp.split(kp.KIND_F16, qkv.to(dev))
    planes = torch.stack([hi, lo])
    return off, planes[0], planes[1]


def _bound_ref(value, r0, S, scale, stream):
    x = value[r0:r0 + S].reshape(S, 3, H, DH)
    q, k, v = x[:, 0], x[:, 1], x[:, 2]
    p = torch.softmax(scale * torch.einsum("ihd,jhd->hij", q, k), dim=-1)
    o = torch.einsum("hij,jhd->ihd", p, v)
    scale_o = torch.einsum("hij,jhd->ihd", p, v.abs())
    L = (scale * torch.einsum("ihd,jhd->hij", q.abs(), k.abs()).amax(-1)).permute(1, 0)[..., None]  # [S, H, 1]
    if stream:  # test_gpu_long_clips.py's bound of the streaming kernel
        tol = (C_OUT * 2.0 ** -18 + (2.0 * 2.0 ** -20 + 2.0 ** -21) * L + (-(-S // 64)) * 2.0 ** -21) * scale_o
    else:  # test_gpu_attention.py's bound of the 160-key kernel
        tol = (C_OUT * 2.0 ** -18 + 2.0 * 2.0 ** -20 * L) * scale_o
    return o.reshape(S, D), tol.reshape(S, D)


def test_packed_attention_kernels_against_float64(cuda_device):
    """Both wgmma kernels on packed clips, each launch walking its own list of clip indices (out of order): within the
    float64 bounds of the uniform-clip tests, bit-identical to the same clip launched alone, no NaN from the poisoned clip
    in any other, and nothing written outside the listed clips."""
    dev = cuda_device
    pap.lib()
    tokens = SHORT[:3] + LONG[:2] + SHORT[3:] + LONG[2:]
    tokens.insert(UNLISTED_CLIP, 100)
    off, qkv_hi, qkv_lo = _packed(dev, tokens, 3)
    value = kp.pair_value(qkv_hi, qkv_lo)
    rows = qkv_hi.shape[0]
    scale = 1.0 / math.sqrt(DH)
    ctx_hi = torch.full((rows, D), SENTINEL, dtype=torch.float16, device=dev)
    ctx_lo = torch.full((rows, D), SENTINEL, dtype=torch.float16, device=dev)
    clip_off = torch.tensor(off, dtype=torch.int32, device=dev)
    listed = [c for c in range(len(tokens)) if c != UNLISTED_CLIP]
    short = [c for c in listed if tokens[c] <= 160][::-1]
    long_ = [c for c in listed if tokens[c] > 160][::-1]
    for ids, which in ((short, kp.ATTN_WGMMA), (long_, kp.ATTN_WGMMA_STREAM)):
        S = max(tokens[c] for c in ids)
        rc = pap.attention_packed(qkv_hi, qkv_lo, ctx_hi, ctx_lo, clip_off, torch.tensor(ids, dtype=torch.int32, device=dev),
                                 S, D, H, scale, which)
        assert rc == 0, (which, rc)
    torch.cuda.synchronize()
    u0, u1 = off[UNLISTED_CLIP], off[UNLISTED_CLIP + 1]
    assert bool((ctx_hi[u0:u1] == SENTINEL).all()) and bool((ctx_hi[off[-1]:] == SENTINEL).all()), "wrote outside the lists"
    got = kp.pair_value(ctx_hi, ctx_lo)
    for c in listed:
        r0, S = off[c], tokens[c]
        stream = S > 160
        # the same clip alone: rows [0, S) of its own buffer, B = 1
        a_hi = torch.full((S + 37, D), SENTINEL, dtype=torch.float16, device=dev)
        a_lo = a_hi.clone()
        q_hi = torch.full((S + 37, 3 * D), float("nan"), dtype=torch.float16, device=dev)
        q_lo = q_hi.clone()
        q_hi[:S], q_lo[:S] = qkv_hi[r0:r0 + S], qkv_lo[r0:r0 + S]
        which = kp.ATTN_WGMMA_STREAM if stream else kp.ATTN_WGMMA
        assert kp.attention(q_hi, q_lo, a_hi, a_lo, 1, S, D, H, scale, kp.KIND_F16, which) == 0
        torch.cuda.synchronize()
        assert torch.equal(ctx_hi[r0:r0 + S].view(torch.int16), a_hi[:S].view(torch.int16)), f"clip {c} ({S} tokens)"
        assert torch.equal(ctx_lo[r0:r0 + S].view(torch.int16), a_lo[:S].view(torch.int16)), f"clip {c} ({S} tokens)"
        if c == POISONED_CLIP:
            continue
        assert bool(torch.isfinite(got[r0:r0 + S]).all()), f"NaN leaked into clip {c}"
        ref, tol = _bound_ref(value, r0, S, scale, stream)
        ratio = float(((got[r0:r0 + S] - ref).abs() / tol).max())
        assert ratio <= 1.0, f"clip {c} ({S} tokens): max |err| / bound = {ratio:.3f}"
        assert _split_ok(ctx_hi[r0:r0 + S], ctx_lo[r0:r0 + S])


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
class _CountingTape:
    def __init__(self, dev):
        self.calls, self.dev = 0, dev

    def randn(self, *shape, device=None, **kw):
        self.calls += 1
        return torch.randn(*shape).to(self.dev)

    def randn_like(self, x):
        self.calls += 1
        return torch.randn(x.shape).to(self.dev)


def _ragged_batch(dev, B=2, T=16):
    x, cond, ts = _inputs(B, T, 41, dev)
    return {'x_t': x, 'cond': cond, 'lengths': torch.tensor([T, T // 2][:B], device=dev)}, ts


def test_unsupported_configurations_are_refused_before_any_launch(cuda_device):
    """tf32x3 / tf32 precisions and head dim 64: refused before an engine exists (nothing has run on the device)."""
    for prec in (_lib.PRECISION_TF32X3, _lib.PRECISION_TF32):
        m = _model(cuda_device)
        m.precision = prec
        batch, ts = _ragged_batch(cuda_device)
        with pytest.raises(RohmB200Error, match="out of scope"):
            m(batch, ts)
        assert m._engine is None
    m = _model(cuda_device, num_heads=8)
    batch, ts = _ragged_batch(cuda_device)
    with pytest.raises(RohmB200Error, match="head dim 64"):
        m(batch, ts)
    assert m._engine is None


def test_bad_lengths_are_refused_before_any_launch(cuda_device):
    B, T = 2, 16
    bad = [torch.tensor([16.0, 8.0]), torch.tensor([16, 8, 4]), torch.tensor([[16, 8]]), torch.tensor([0, 8]),
           torch.tensor([17, 8]), torch.tensor([16, -1]), torch.tensor([True, True]), [16, 8]]
    for lengths in bad:
        m = _model(cuda_device)
        batch, ts = _ragged_batch(cuda_device, B, T)
        batch['lengths'] = lengths.to(cuda_device) if isinstance(lengths, torch.Tensor) else lengths
        with pytest.raises(RohmB200Error, match="lengths"):
            m(batch, ts)
        assert m._engine is None, lengths


def test_prox_and_global_guidance_are_refused_before_any_launch(cuda_device):
    B, T = 2, 16
    m = _model(cuda_device)
    batch, _ = _ragged_batch(cuda_device, B, T)
    del batch['x_t']
    d = _diff(cuda_device)
    tape = _CountingTape(cuda_device)
    d._randn, d._randn_like = tape.randn, tape.randn_like
    with pytest.raises(RohmB200Error, match="prox"):
        d.p_sample_loop(m, batch, [B, 294, 1, T], clip_denoised=False, cond_fn_with_grad=True, grad_type='prox')
    m.guidance_sum_reducer = lambda s: s
    with pytest.raises(RohmB200Error, match="global_guidance"):
        d.p_sample_loop(m, batch, [B, 294, 1, T], clip_denoised=False, cond_fn_with_grad=True, grad_type='amass')
    assert tape.calls == 0 and m._engine is None
    x = torch.zeros(B, 294, 1, T, device=cuda_device)
    with pytest.raises(RohmB200Error, match="global_guidance"):
        m.guide_skating_with_smpl(batch, {'pred_xstart': x}, None, compute_grad='x_0')
    del m.guidance_sum_reducer
    with pytest.raises(RohmB200Error, match="prox"):
        m.guide_2d_projection_with_smpl(batch, {'pred_xstart': x}, None, compute_grad='x_0')
