"""TrajNet and TrajNet + TrajControl on batches of clips with different lengths (batch['lengths']): every clip's frames
depend on that clip alone, bit for bit, and match the clip at its own length up to summation order; padded frames are zero
and their inputs never matter; the packed GroupNorm and GEMM row mask through the kernel probe; and the refusals."""
import argparse

import pytest
import torch

import kernel_probe as kp
from helpers import TOL
from oracle import trajnet_oracle
from rohm_b200 import _lib, diffusion, synthetic
from rohm_b200._lib import RohmB200Error
from rohm_b200.trajnet import TrajNet
from test_gpu_long_trajnet import SENTINEL, _gn_reference

pytestmark = pytest.mark.gpu

LENGTHS, T_RAGGED = [2000, 1536, 1008, 144, 16], 2000  # 1- and 2-CTA GroupNorm clusters, the shortest legal clip


def _build(control, dev, seed=2):
    m = TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=control, device=dev,
                dataset=synthetic.make_dataset('traj'), repr_abs_only=True)
    sd = {k: v.cpu() for k, v in synthetic.synth_state_dict(m, seed).items()}
    m.load_state_dict(sd)
    return m.to(dev).eval(), sd


@pytest.fixture(scope="module")
def nets(cuda_device):
    return {False: _build(False, cuda_device), True: _build(True, cuda_device)}


def _inputs(B, T, control, seed, dev):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, 13, generator=gen)
    batch = {k: v.to(dev) for k, v in synthetic.trajnet_batch(B, T, seed, control=control).items() if k != 'motion_repr_clean'}
    batch['x_t'] = x.to(dev)
    ts = torch.randint(0, 1000, (B,), generator=gen).to(dev)
    return batch, ts


def _bits(t):
    return t.contiguous().view(torch.int32)


def _poison(t, lengths):
    """A copy with every padded frame filled with NaN, +Inf, -Inf and 1e30 in turn."""
    t = t.clone()
    vals = torch.tensor([float("nan"), float("inf"), float("-inf"), 1e30], device=t.device)
    T = t.shape[1]
    for b, n in enumerate(lengths):
        if n < T:
            t[b, n:] = vals[torch.arange(n, T, device=t.device) % 4].view(-1, 1)
    return t


def _clip(batch, b, n=None, lengths=True):
    """Clip b of a batch: padded to the batch's T with its length, or (n given) cut to its first n frames without it."""
    keys = ('x_t', 'cond', 'control_cond')
    out = {k: (batch[k][b:b + 1] if n is None else batch[k][b:b + 1, :n]).contiguous() for k in keys if k in batch}
    if n is None and lengths:
        out['lengths'] = batch['lengths'][b:b + 1]
    return out


_ORACLE = {}


@pytest.mark.parametrize("prec", [_lib.PRECISION_F16X2, _lib.PRECISION_TF32X3])
@pytest.mark.parametrize("control", [False, True])
def test_ragged_forward(nets, cuda_device, control, prec):
    """Each clip bit-identical to itself as a one-clip padded batch through the same engine and after a permutation of
    the clips; within 2e-5 max(1, scale) of the clip at its own length, both within TOL of the oracle on the clip alone;
    padded frames exactly zero; the same bits with NaN, +-Inf and 1e30 in the padded frames of every input."""
    m, sd = nets[control]
    m.precision = prec
    try:
        B, T = len(LENGTHS), T_RAGGED
        batch, ts = _inputs(B, T, control, 3, cuda_device)
        batch['lengths'] = torch.tensor(LENGTHS, device=cuda_device)
        out = m(batch, ts).clone()
        e = m._engine
        for b, n in enumerate(LENGTHS):
            assert bool((out[b, n:] == 0).all()), f"clip {b}: padded frames are not zero"
            one = m(_clip(batch, b), ts[b:b + 1])
            assert m._engine is e, "a one-clip batch of the same T must reuse the engine"
            assert torch.equal(_bits(one), _bits(out[b:b + 1])), f"clip {b} ({n} frames) depends on other clips"
        perm = [3, 0, 4, 2, 1]
        pb = {k: v[perm].contiguous() for k, v in batch.items()}
        outp = m(pb, ts[perm])
        assert torch.equal(_bits(outp), _bits(out[perm])), "clip order changed a result"
        poisoned = {k: (_poison(v, LENGTHS) if k != 'lengths' else v) for k, v in batch.items()}
        assert torch.equal(_bits(m(poisoned, ts)), _bits(out)), "values in padded frames reached a real frame"
        for b, n in enumerate(LENGTHS):
            own = m(_clip(batch, b, n), ts[b:b + 1])
            scale = max(1.0, float(own.abs().max()))
            assert float((out[b, :n] - own[0]).abs().max()) <= 2e-5 * scale, (b, n)
            key = (control, b)
            if key not in _ORACLE:
                cb = {k: v.cpu() for k, v in _clip(batch, b, n).items()}
                with torch.no_grad():
                    _ORACLE[key] = trajnet_oracle.trajnet_forward(sd, cb['x_t'], cb['cond'], ts[b:b + 1].cpu(),
                                                                  cb.get('control_cond'))
            ref = _ORACLE[key]
            assert float((out[b, :n].cpu() - ref[0]).abs().max()) < TOL, (b, n)
            assert float((own[0].cpu() - ref[0]).abs().max()) < TOL, (b, n)
    finally:
        m.precision = None


@pytest.mark.parametrize("B,T", [(64, 144), (3, 1536)])
def test_uniform_lengths_equal_no_lengths(nets, cuda_device, B, T):
    """lengths = T for every clip gives the bits of the batch without the key; so does a forward without the key after
    one with it (the engine returns to uniform clips)."""
    m, _ = nets[True]
    batch, ts = _inputs(B, T, True, 20 + T, cuda_device)
    ref = m(batch, ts).clone()
    got = m(dict(batch, lengths=torch.full((B,), T, dtype=torch.int32, device=cuda_device)), ts).clone()
    assert torch.equal(_bits(got), _bits(ref))
    again = m(batch, ts)
    assert torch.equal(_bits(again), _bits(ref))


class _SlicedTape:
    """Seeded noise for a padded [B, T, 13] batch, draw by draw; with clip=(b, n) every draw is the slice [b:b+1, :n] of
    the same padded draw (n = None: the clip padded to T)."""

    def __init__(self, seed, full_shape, device, clip=None):
        self.seed, self.full, self.device, self.clip, self.k = seed, tuple(full_shape), device, clip, 0

    def _draw(self, shape):
        z = torch.randn(self.full, generator=torch.Generator().manual_seed(1000 * self.seed + self.k))
        self.k += 1
        if self.clip is not None:
            b, n = self.clip
            z = z[b:b + 1] if n is None else z[b:b + 1, :n]
        assert tuple(z.shape) == tuple(shape), (z.shape, shape)
        return z.contiguous().to(self.device)

    def randn(self, *shape, device=None, **kw):
        return self._draw(shape)

    def randn_like(self, x):
        return self._draw(x.shape)


def _diff(dev, steps='20'):
    a = argparse.Namespace(noise_schedule='cosine', sigma_small=True)
    return diffusion.create_gaussian_diffusion(a, diffusion, diffusion.SpacedDiffusionTrajNet, 1000, steps, dev)


def _taped(dev, tape):
    d = _diff(dev)
    d._randn, d._randn_like = tape.randn, tape.randn_like
    return d


def test_ragged_sampling(nets, cuda_device):
    """A 20-step respaced p_sample_loop over a ragged TrajControl batch, noise injected through the diffusion object's
    hooks: every clip bit-identical to its loop as a one-clip padded batch, within TOL of its loop at its own length, and
    the final sample's padded frames zero."""
    m, _ = nets[True]
    lengths = [2000, 1008, 144, 16]
    B, T = len(lengths), 2000
    shape = (B, T, 13)
    batch, _ = _inputs(B, T, True, 31, cuda_device)
    del batch['x_t']
    batch['lengths'] = torch.tensor(lengths, device=cuda_device)
    out = _taped(cuda_device, _SlicedTape(5, shape, cuda_device)).p_sample_loop(m, dict(batch), list(shape),
                                                                                clip_denoised=False)
    e = m._engine
    for b, n in enumerate(lengths):  # before any clip at its own length: that rebuilds the engine for another T
        assert bool((out[b, n:] == 0).all()), f"clip {b}: padded frames of the final sample are not zero"
        d1 = _taped(cuda_device, _SlicedTape(5, shape, cuda_device, clip=(b, None)))
        padded = d1.p_sample_loop(m, _clip(batch, b), [1, T, 13], clip_denoised=False)
        assert m._engine is e, "a one-clip batch of the same T must reuse the engine"
        assert torch.equal(_bits(out[b:b + 1]), _bits(padded)), f"clip {b} ({n} frames)"
    for b, n in enumerate(lengths):
        d2 = _taped(cuda_device, _SlicedTape(5, shape, cuda_device, clip=(b, n)))
        own = d2.p_sample_loop(m, _clip(batch, b, n), [1, n, 13], clip_denoised=False)
        assert float((out[b:b + 1, :n] - own).abs().max()) < TOL, (b, n)


def _loop(m, batch, shape, dev, seed=77):
    torch.manual_seed(seed)
    return _diff(dev, '').p_sample_loop(m, dict(batch), list(shape), clip_denoised=False)


def test_graph_variants_under_lengths(cuda_device, monkeypatch):
    """Under lengths, bit for bit: the fused sample step against the unfused chain, the serial forward graph against
    the multi-stream one, and eager launches against graph replay."""
    lengths = [1536, 144, 16]
    B, T = len(lengths), 1536
    batch, ts = _inputs(B, T, True, 9, cuda_device)
    batch['lengths'] = torch.tensor(lengths, device=cuda_device)
    gen = torch.cuda.default_generators[cuda_device.index]
    m, _ = _build(True, cuda_device)
    sample_batch = {k: v for k, v in batch.items() if k != 'x_t'}
    outs, offs = [], []
    d = diffusion.create_gaussian_diffusion(argparse.Namespace(noise_schedule='cosine', sigma_small=True), diffusion,
                                            diffusion.SpacedDiffusionTrajNet, 4, '', cuda_device)
    for fused in (True, False):
        monkeypatch.setattr(diffusion, "_FUSED_STEP", fused)
        torch.manual_seed(77)
        outs.append(d.p_sample_loop(m, dict(sample_batch), [B, T, 13], clip_denoised=False))
        offs.append(gen.get_offset())
    assert torch.equal(_bits(outs[0]), _bits(outs[1])) and offs[0] == offs[1]
    for b, n in enumerate(lengths):
        assert bool((outs[0][b, n:] == 0).all())
    ref = m(batch, ts).clone()
    monkeypatch.setenv("ROHM_B200_TRAJ_PARALLEL", "0")
    m_ser, _ = _build(True, cuda_device)
    assert torch.equal(_bits(m_ser(batch, ts)), _bits(ref)), "serial graph differs from the multi-stream graph"
    monkeypatch.delenv("ROHM_B200_TRAJ_PARALLEL")
    monkeypatch.setenv("ROHM_B200_GRAPH", "0")
    m_eager, _ = _build(True, cuda_device)
    assert torch.equal(_bits(m_eager(batch, ts)), _bits(ref)), "eager launches differ from the graph"


def test_changing_lengths_between_calls(nets, cuda_device):
    """A new lengths tensor, and the same tensor edited in place: the new lengths are used and the condition is
    re-embedded (the reference runs use fresh condition tensors, which always embed)."""
    m, _ = nets[True]
    B, T = 3, 1536
    batch, ts = _inputs(B, T, True, 13, cuda_device)
    la, lb = [1536, 512, 16], [144, 1536, 1008]

    def fresh(lengths):
        fb = {k: v.clone() for k, v in batch.items()}
        fb['lengths'] = torch.tensor(lengths, device=cuda_device)
        return m(fb, ts).clone()

    ref_a, ref_b = fresh(la), fresh(lb)
    assert not torch.equal(ref_a, ref_b)
    L = torch.tensor(la, device=cuda_device)
    assert torch.equal(_bits(m(dict(batch, lengths=L), ts)), _bits(ref_a))
    assert torch.equal(_bits(m(dict(batch, lengths=torch.tensor(lb, device=cuda_device)), ts)), _bits(ref_b))
    assert torch.equal(_bits(m(dict(batch, lengths=L), ts)), _bits(ref_a))
    L.copy_(torch.tensor(lb, device=cuda_device))
    assert torch.equal(_bits(m(dict(batch, lengths=L), ts)), _bits(ref_b))


# ---------------------------------------------------------------------------------------------------------------------
# the packed GroupNorm and GEMM row mask through the kernel probe
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,div", [(64, 1), (512, 16)])
def test_packed_group_norm_matches_float64(cuda_device, C, div):
    """gn_mish_split_kernel with a packed offset table (engine T = 1536, clusters of 1 and 2, clips shorter than one
    slice): each clip within the float64 bound of _gn_reference on that clip alone, its pad rows zero, nothing written
    past the packed matrix, and bit-identical to the clip launched alone as a one-clip packed batch."""
    T, lengths = 1536, [1536, 16, 1008, 144]
    L = div.bit_length() - 1
    TL, Tp = T >> L, (T + 32) >> L
    off = [0]
    for n in lengths:
        off.append(off[-1] + ((n + 32) >> L))
    B, rows = len(lengths), off[-1]
    gen = torch.Generator().manual_seed(C + div)
    rnd = lambda *s: torch.randn(*s, generator=gen).to(cuda_device)
    for splits, extras, f16 in ((1, False, 1), (3, True, 1), (8, True, 0)):
        part = rnd(splits, rows * C)
        bias, gamma, beta = rnd(C) * 0.5, 1.0 + 0.2 * rnd(C), 0.3 * rnd(C)
        tp = rnd(B, C + 4) if extras else None
        r1 = rnd(rows * C) if extras else None
        r2 = rnd(rows * C) if extras else None
        pair_dtype = torch.float16 if f16 else torch.float32

        def run(n, clip_off, nb, part_, tp_, r1_, r2_, nrows):
            extra = 64
            out = torch.full((nrows * C + extra,), SENTINEL, device=cuda_device)
            hi = torch.full((nrows * C + extra,), SENTINEL, device=cuda_device, dtype=pair_dtype)
            lo = torch.full_like(hi, SENTINEL)
            rc = kp.group_norm(part_, splits, part_.shape[1], bias, gamma, beta, tp_, C + 4, r1_, r2_, out, hi, lo, C, Tp, TL, nb,
                               n, f16, clip_off=torch.tensor(clip_off, dtype=torch.int32, device=cuda_device))
            torch.cuda.synchronize()
            assert rc == 0, rc
            for buf in (out, hi, lo):
                assert bool((buf[nrows * C:].float() == SENTINEL).all()), (n, "wrote past the packed matrix")
            return out

        for n in (1, 2):
            out = run(n, off, B, part, tp, r1, r2, rows)
            for b, ln in enumerate(lengths):
                r0, rb, tb = off[b], off[b + 1] - off[b], ln >> L
                sl = lambda t: None if t is None else t[r0 * C:(r0 + rb) * C].contiguous()
                ref, bound = _gn_reference([p[r0 * C:(r0 + rb) * C] for p in part], bias, gamma, beta,
                                           None if tp is None else tp[b:b + 1], sl(r1), sl(r2), 1, rb, tb, C)
                o = out[r0 * C:(r0 + rb) * C].view(rb, C)
                assert bool((o[tb:] == 0).all()), (n, b, "pad rows must be zero")
                err = (o[:tb].double() - ref[0]).abs()
                assert bool((err <= bound[0]).all()), (n, b, float(err.max()))
                alone = run(n, [0, rb], 1, part[:, r0 * C:(r0 + rb) * C].contiguous(),
                            None if tp is None else tp[b:b + 1].contiguous(), sl(r1), sl(r2), rb)
                assert torch.equal(alone[:rb * C], out[r0 * C:(r0 + rb) * C]), (n, b)


@pytest.mark.parametrize("tma", [False, True])
def test_gemm_row_mask(cuda_device, tma):
    """The masked GEMM epilogue with a packed row mask: masked rows are exactly zero, the others bit-identical to the same
    launch with every row real, and nothing is written past M."""
    kind, M, K, N = kp.KIND_F16, 300, 64, 64
    gen = torch.Generator().manual_seed(4)
    a = torch.randn(M, K, generator=gen).to(cuda_device)
    w = torch.randn(N, K, generator=gen).to(cuda_device) * 0.1
    bias = torch.randn(N, generator=gen).to(cuda_device)
    A, W = kp.Operand(kind, a), kp.Weight(kind, [w], 64)
    mask = (torch.rand(M, generator=gen) < 0.6).to(torch.uint8).to(cuda_device)
    outs = []
    for rm in (None, mask):
        out = torch.full((M + 8, N), SENTINEL, device=cuda_device)
        rc, g = kp.gemm(kind, W, [A.seg(W.kblocks[0])], M, N, out=out, bias=bias, act=kp.ACT_MISH, clip_rows=M, clip_valid=M,
                        row_mask=rm, tma_store=tma)
        torch.cuda.synchronize()
        assert rc == 0, rc
        assert g.tma_store == int(tma), "the bulk-store epilogue was not taken as asked"
        assert bool((out[M:] == SENTINEL).all())
        outs.append(out[:M])
    full, masked = outs
    keep = mask.bool()
    assert bool((masked[~keep] == 0).all())
    assert torch.equal(_bits(masked[keep]), _bits(full[keep]))
    assert float(full[keep].abs().max()) > 0


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


def test_bad_lengths_are_refused_before_any_launch(cuda_device):
    """Wrong dtype, shape or type, out of range and not a multiple of 16: refused by the forward and by every sampling
    loop before an engine exists or a noise draw happens."""
    B, T = 2, 32
    bad = [torch.tensor([32.0, 16.0]), torch.tensor([32, 16, 16]), torch.tensor([[32, 16]]), torch.tensor([0, 16]),
           torch.tensor([48, 16]), torch.tensor([32, 8]), torch.tensor([32, 24]), torch.tensor([32, -16]),
           torch.tensor([True, True]), [32, 16]]
    for lengths in bad:
        m, _ = _build(True, cuda_device)
        batch, ts = _inputs(B, T, True, 41, cuda_device)
        batch['lengths'] = lengths.to(cuda_device) if isinstance(lengths, torch.Tensor) else lengths
        with pytest.raises(RohmB200Error, match="lengths"):
            m(batch, ts)
        del batch['x_t']
        for steps in ('4', 'ddim4'):
            d = _diff(cuda_device, steps)
            tape = _CountingTape(cuda_device)
            d._randn, d._randn_like = tape.randn, tape.randn_like
            with pytest.raises(RohmB200Error, match="lengths"):
                if steps.startswith('ddim'):
                    d.ddim_sample_loop(m, dict(batch), [B, T, 13], clip_denoised=False)
                else:
                    d.p_sample_loop(m, dict(batch), [B, T, 13], clip_denoised=False)
            assert tape.calls == 0, (lengths, steps)
        assert m._engine is None, lengths


def test_losses_with_lengths_are_refused_before_any_launch(cuda_device):
    B, T = 2, 32
    m, _ = _build(True, cuda_device)
    batch, _ = _inputs(B, T, True, 43, cuda_device)
    del batch['x_t']
    batch['lengths'] = torch.tensor([32, 16], device=cuda_device)
    d = _diff(cuda_device, '4')
    tape = _CountingTape(cuda_device)
    d._randn, d._randn_like = tape.randn, tape.randn_like
    with pytest.raises(RohmB200Error, match="compute_loss=False"):
        d.eval_losses(m, batch, [B, T, 13], clip_denoised=False, compute_loss=True)
    assert tape.calls == 0 and m._engine is None
    _, out = d.eval_losses(m, batch, [B, T, 13], clip_denoised=False, compute_loss=False)
    assert bool((out[1, 16:] == 0).all())
