"""Clip sharding across the GPUs of one box.

Every tensor on the hot path has the clip as its leading dimension and nothing in either denoiser mixes clips
(SURVEY.md 8e), so the batch is split into contiguous per-rank shards, each rank runs the unmodified single-GPU loop on
its shard with a full replica of the weights, and ONE NCCL all-gather of the final per-clip outputs reassembles the
batch (no intra-step collective).  Guidance is the one batch-coupled piece (the skating loss is normalised by a
batch-wide count): per-shard semantics are the contract, i.e. each shard equals the reference run on that sub-batch.

Noise: in parity mode the full-batch tensor is drawn from the global generator on every rank and sliced, so the
concatenated result is bit-identical to the single-GPU run with the same seed.
"""
import torch
import torch.distributed as dist


def shard_bounds(n_clips, rank, world):
    """Contiguous split; the first n_clips % world ranks get one extra clip."""
    base, extra = divmod(int(n_clips), int(world))
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_batch(batch, rank, world, n_clips=None):
    """Slices every tensor whose leading dim equals the global batch size; other entries are passed through."""
    if n_clips is None:
        n_clips = max(v.shape[0] for v in batch.values() if torch.is_tensor(v) and v.dim() > 0)
    lo, hi = shard_bounds(n_clips, rank, world)
    return {k: (v[lo:hi] if torch.is_tensor(v) and v.dim() > 0 and v.shape[0] == n_clips else v) for k, v in batch.items()}


class ShardedNoise:
    """randn / randn_like replacements that reproduce the single-process random stream: draw the FULL-batch tensor
    (same generator, same order, same shapes as the unsharded run) and return this rank's slice."""

    def __init__(self, n_clips, rank, world, generator=None):
        self.n, self.rank, self.world, self.generator = int(n_clips), rank, world, generator
        self.lo, self.hi = shard_bounds(n_clips, rank, world)

    def randn(self, *shape, device=None, **kw):
        shape = list(shape[0]) if len(shape) == 1 and isinstance(shape[0], (list, tuple)) else list(shape)
        full = torch.randn([self.n] + shape[1:], device=device, generator=self.generator)
        return full[self.lo:self.hi].contiguous()

    def randn_like(self, x):
        full = torch.randn([self.n] + list(x.shape[1:]), device=x.device, dtype=x.dtype, generator=self.generator)
        return full[self.lo:self.hi].contiguous()

    def install(self, diffusion):
        diffusion._randn, diffusion._randn_like = self.randn, self.randn_like
        return diffusion


def gather_clips(local_out, n_clips, group=None):
    """The single collective of the path: all ranks receive the [n_clips, ...] tensor of final outputs.
    One all_gather_into_tensor (NCCL all-gather over NVLink); ragged shards are padded to the largest shard first."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    sizes = [shard_bounds(n_clips, r, world)[1] - shard_bounds(n_clips, r, world)[0] for r in range(world)]
    assert local_out.shape[0] == sizes[rank], (local_out.shape, sizes, rank)
    if len(set(sizes)) == 1:
        out = torch.empty([n_clips] + list(local_out.shape[1:]), dtype=local_out.dtype, device=local_out.device)
        dist.all_gather_into_tensor(out, local_out.contiguous(), group=group)
        return out
    # ragged shards: pad every shard to the largest one, gather once, drop the padding
    mx = max(sizes)
    padded = torch.zeros([mx] + list(local_out.shape[1:]), dtype=local_out.dtype, device=local_out.device)
    padded[:sizes[rank]] = local_out
    buf = torch.empty([world * mx] + list(local_out.shape[1:]), dtype=local_out.dtype, device=local_out.device)
    dist.all_gather_into_tensor(buf, padded, group=group)
    return torch.cat([buf[r * mx: r * mx + sizes[r]] for r in range(world)], dim=0)


def global_guidance(model, group=None, enable=True):
    """Guidance normalisers of a clip-sharded run.  Default contract (enable=False): each shard equals the reference run on
    that sub-batch.  enable=True: the skating loss is normalised by the batch-wide counts as in an unsharded reference run --
    one 4-float all-reduce per guided step (the only intra-step collective of the path; <= 51 of 1000 steps), which makes the
    gathered result reproduce the single-GPU run on the whole batch.  Refused for a model in guidance_normaliser='clip'
    mode: each clip is then normalised by its own counts, which needs no collective."""
    if not enable:
        if hasattr(model, "guidance_sum_reducer"):
            del model.guidance_sum_reducer
        return model
    if getattr(model, "guidance_normaliser", "batch") == "clip":
        from ._lib import RohmB200Error
        raise RohmB200Error("global_guidance: the model normalises its guidance per clip (guidance_normaliser='clip'), "
                            "which needs no collective and contradicts the batch-wide normaliser")
    model.guidance_sum_reducer = lambda sums: dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=group)
    return model


def shard_generators(generators, rank, world):
    """This rank's slice of the global batch's per-clip generators (batch['generators']), by shard_bounds."""
    lo, hi = shard_bounds(len(generators), rank, world)
    return list(generators[lo:hi])


def sample_sharded(diffusion, model, batch, shape, parity_noise=True, group=None, **eval_kwargs):
    """eval_losses on this rank's shard + the final all-gather.  `batch` and `shape` describe the GLOBAL batch.
    With batch['generators'] (one CUDA generator per clip, rohm_b200.noise_streams) each rank gets its slice of the list
    and draws only its own clips' noise; no ShardedNoise is installed, so the fused step graph stays on."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    n = int(shape[0])
    local = shard_batch(batch, rank, world, n)
    lo, hi = shard_bounds(n, rank, world)
    lshape = [hi - lo] + list(shape[1:])
    if batch.get('generators') is not None:
        local['generators'] = shard_generators(batch['generators'], rank, world)
        parity_noise = False  # each clip's noise comes from its own generator, wherever it runs
    if parity_noise:
        ShardedNoise(n, rank, world).install(diffusion)
    try:
        _, out = diffusion.eval_losses(model=model, batch=local, shape=lshape, compute_loss=False, **eval_kwargs)
    finally:
        if parity_noise:
            diffusion._randn, diffusion._randn_like = torch.randn, torch.randn_like
    return gather_clips(out, n, group)
