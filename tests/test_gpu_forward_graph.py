"""Replays of the engines' cached forward graphs (rohm_b200/csrc/graph.cu) with caller buffers that are all alive at distinct
addresses, so a replay that kept a captured pointer would read or write the wrong tensor.  Every result must equal the same
engine's eager launches (rohm_*_set_option(0, 0)) bit for bit."""
import pytest
import torch

from rohm_b200 import synthetic, trajnet_engine
from rohm_b200.posenet import PoseNet
from rohm_b200.trajnet import TrajNet

pytestmark = pytest.mark.gpu


class _PoseNetCase:
    B, T = 2, 16

    def __init__(self, dev):
        m = PoseNet(dataset=synthetic.make_dataset('pose'), body_feat_dim=294, latent_dim=512, ff_size=1024, num_layers=8,
                    num_heads=4, device=dev, traj_feat_dim=22)
        m.load_state_dict(synthetic.synth_state_dict(m, 1))
        self.m, self.dev = m.to(dev).eval(), dev

    def engine(self, T=None):
        """A new engine (an empty graph cache) holding the condition of T frames."""
        self.m.invalidate_engine()
        return self.set_cond(T or self.T)

    def set_cond(self, T):
        return self.m.prepare_cond(synthetic.posenet_batch(self.B, T, 5 + T)['cond'].to(self.dev))

    def inputs(self, seed, T=None):
        gen = torch.Generator().manual_seed(seed)
        x = torch.randn(self.B, 294, 1, T or self.T, generator=gen)
        return x.to(self.dev), torch.randint(0, 1000, (self.B,), generator=gen).to(self.dev)

    def forward(self, e, x, t):
        return e.forward(x, t, torch.empty_like(x))

    def graphs(self, e, on):
        assert e.lib.rohm_posenet_set_option(e.handle, 0, int(on)) == 0


class _TrajControlCase:
    B, T = 3, 144

    def __init__(self, dev):
        m = TrajNet(time_dim=32, mid_dim=512, cond_dim=13, traj_feat_dim=13, trajcontrol=True, device=dev,
                    dataset=synthetic.make_dataset('traj'), repr_abs_only=True)
        m.load_state_dict(synthetic.synth_state_dict(m, 2))
        self.m, self.dev = m.to(dev).eval(), dev
        self.batch = {k: v.to(dev) for k, v in synthetic.trajnet_batch(self.B, self.T, 9, control=True).items()}

    def engine(self):
        self.m._engine = None
        self.batch['x_t'] = torch.zeros(self.B, self.T, 13, device=self.dev)
        e, _, _ = trajnet_engine.prepare(self.m, self.batch, torch.zeros(self.B, dtype=torch.int64, device=self.dev))
        return e

    def inputs(self, seed):
        gen = torch.Generator().manual_seed(seed)
        x = torch.randn(self.B, self.T, 13, generator=gen)
        return x.to(self.dev), torch.randint(0, 1000, (self.B,), generator=gen).to(self.dev)

    def forward(self, e, x, t):
        return e._forward_impl(x, t)

    def graphs(self, e, on):
        assert e.lib.rohm_trajnet_set_option(e.handle, 0, int(on)) == 0


@pytest.fixture(scope="module", params=["posenet", "trajcontrol"])
def case(request, cuda_device):
    return (_PoseNetCase if request.param == "posenet" else _TrajControlCase)(cuda_device)


def test_replay_takes_every_caller_pointer_of_the_call(case):
    """Capture with (x1, t1, out1), then replay with (x2, t2, out2): out2 is the eager forward of (x2, t2), and out1 still
    holds the first result."""
    e = case.engine()
    (x1, t1), (x2, t2) = case.inputs(1), case.inputs(2)
    out1 = case.forward(e, x1, t1)  # captures the graph, then replays it
    first = out1.clone()
    out2 = case.forward(e, x2, t2)
    case.graphs(e, False)
    ref1, ref2 = case.forward(e, x1, t1), case.forward(e, x2, t2)
    case.graphs(e, True)
    assert torch.equal(out2, ref2)
    assert torch.equal(out1, first) and torch.equal(first, ref1)


def test_replayed_sample_step_takes_every_argument_of_the_call(case):
    """Two fused steps (forward + in-kernel-noise update) with their own x_t, timesteps, coefficient row and generator state
    (seed, offset): pred_xstart, x_{t-1} and the generator's offset afterwards equal the eager launches'."""
    e = case.engine()
    gen = torch.cuda.default_generators[case.dev.index]
    calls = []
    for seed, offset in ((11, 0), (12, 64)):
        x, t = case.inputs(seed)
        coef = torch.rand(8, generator=torch.Generator().manual_seed(seed)).to(case.dev)
        calls.append((x, t, coef, seed, offset))

    def run():
        results = []
        for x, t, coef, seed, offset in calls:
            gen.manual_seed(seed)
            gen.set_offset(offset)
            x0, nxt = e.sample_step(x, t, coef)
            results.append((x0, nxt, gen.get_offset()))
        return results

    graphed = run()  # the first call captures the graph, the second replays it
    case.graphs(e, False)
    eager = run()
    case.graphs(e, True)
    for (g0, gn, goff), (e0, en, eoff) in zip(graphed, eager):
        assert torch.equal(g0, e0) and torch.equal(gn, en) and goff == eoff


def test_evicted_graph_is_captured_again(cuda_device):
    """Nine clip lengths fill the cache of eight graphs and evict the first; its length is then captured again.  The
    lengths descend so that one engine serves them all (PoseNet.engine rebuilds it when T grows)."""
    case = _PoseNetCase(cuda_device)
    lengths = [40, 36, 32, 28, 24, 20, 16, 12, 8, 40]
    e = case.engine(lengths[0])
    for i, T in enumerate(lengths):
        assert case.set_cond(T) is e
        x, t = case.inputs(100 + i, T)
        out = case.forward(e, x, t)
        case.graphs(e, False)
        ref = case.forward(e, x, t)
        case.graphs(e, True)
        assert torch.equal(out, ref), T
