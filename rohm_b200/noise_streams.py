"""Per-clip noise streams: ``batch['generators']``, one ``torch.Generator`` per clip.

With the key, every draw of the samplers gives clip b exactly ``torch.randn(S_b, generator=generators[b])`` for the shape
S_b the clip has when it runs alone (PoseNet ``[1, C, 1, n_b]``, TrajNet ``[1, n_b, C]``, n_b = lengths[b] or T), in its
real frames, and zero in its padded frames.  A recording's noise then depends on the recording and its generator only,
not on the batch it lands in, its position, the padding or the GPU.

The draws run in the library's own kernels (rohm_randn_clips, rohm_ddpm_step_philox_clips and the engines'
*_sample_step_clips), which reproduce torch's Philox ``normal_`` per clip.  The host reads each generator's (seed, offset)
once per loop, uploads them as one table, passes a draw index per step, and writes the offsets back at the end, so they
advance exactly as torch would have advanced them for the same draws.
"""
import ctypes as C

import torch

from ._lib import RohmB200Error

MAX_CLIPS = 256  # rohm_randn_clips: the per-clip launch plan is a kernel parameter


def check_generators(batch, n_clips, device, diffusion=None, const_noise=False):
    """batch['generators'] checked against a batch of `n_clips` clips on `device`: -> the list, or None without the key.
    Raises RohmB200Error before anything runs on the device: wrong count, non-generators, the same generator twice,
    CPU or other-device generators, more than MAX_CLIPS clips, const_noise=True (one noise for every clip), and a
    diffusion whose _randn / _randn_like has been replaced (a recorded tape, parallel.ShardedNoise): two noise sources."""
    gens = batch.get('generators') if isinstance(batch, dict) else None
    if gens is None:
        return None
    if const_noise:
        raise RohmB200Error("batch['generators'] with const_noise=True: const_noise shares clip 0's noise with every clip, "
                            "per-clip streams give every clip its own")
    if diffusion is not None and (diffusion._randn is not torch.randn or diffusion._randn_like is not torch.randn_like):
        raise RohmB200Error("batch['generators'] with a replaced noise source (diffusion._randn / _randn_like, e.g. a "
                            "recorded tape or parallel.ShardedNoise): the two noise sources would be ambiguous")
    if not isinstance(gens, (list, tuple)):
        raise RohmB200Error(f"batch['generators'] must be a list or tuple of torch.Generator, got {type(gens).__name__}")
    if len(gens) != int(n_clips):
        raise RohmB200Error(f"batch['generators'] holds {len(gens)} generators for a batch of {int(n_clips)} clips")
    if len(gens) > MAX_CLIPS:
        raise RohmB200Error(f"batch['generators']: at most {MAX_CLIPS} clips per batch draw from per-clip streams")
    bad = [i for i, g in enumerate(gens) if not isinstance(g, torch.Generator)]
    if bad:
        raise RohmB200Error(f"batch['generators'][{bad[0]}] is a {type(gens[bad[0]]).__name__}, not a torch.Generator")
    if len({id(g) for g in gens}) != len(gens):
        raise RohmB200Error("batch['generators']: the same generator object appears twice; give every clip its own")
    dev = torch.device(device)
    for i, g in enumerate(gens):
        if g.device.type != 'cuda':
            raise RohmB200Error(f"batch['generators'][{i}] is a {g.device.type} generator; the streams are drawn on the "
                                f"batch's CUDA device, so each generator must be torch.Generator(device={str(dev)!r})")
        if dev.type == 'cuda' and dev.index is not None and g.device.index is not None and g.device.index != dev.index:
            raise RohmB200Error(f"batch['generators'][{i}] lives on {g.device}, the batch on {dev}")
    return list(gens)


def _as_i64(v):
    v = int(v)
    return v - (1 << 64) if v >= (1 << 63) else v


class NoiseStreams:
    """The streams of B CUDA generators for one sampling loop or one direct step.  Reads every generator's (seed, offset)
    once, uploads them as a device table int64 [B, 2] (the bits of uint64), and hands out draw indices; draw k of clip b
    starts at offset_b + k * inc_b, inc_b being what torch advances the offset by for that clip's draw.  close() sets each
    generator's offset to where torch would have left it.  Every draw of one NoiseStreams has the same layout."""

    def __init__(self, generators, device):
        self.generators = list(generators)
        self.start = [int(g.get_offset()) for g in self.generators]
        rows = [[_as_i64(g.initial_seed()), _as_i64(o)] for g, o in zip(self.generators, self.start)]
        self.table = torch.tensor(rows, dtype=torch.int64).to(device, non_blocking=False)
        self.incs = (C.c_uint64 * len(self.generators))()  # written by every draw; the same for every draw of a layout
        self.draws = 0
        self._layout = None
        self._lengths_c = None

    def __len__(self):
        return len(self.generators)

    def next_draw(self, layout):
        """The index of the next draw of `layout` = (C, T, channels_last, lengths tuple or None)."""
        if self._layout is None:
            self._layout = layout
        elif layout is not self._layout and layout != self._layout:
            raise RohmB200Error(f"per-clip noise streams: a draw of layout {layout[:3]} after draws of {self._layout[:3]} "
                                "(one loop draws one shape)")
        d = self.draws
        self.draws += 1
        return d

    def lengths_c(self, lengths):
        """`lengths` as a ctypes int array (cached), or None."""
        if lengths is None:
            return None
        if self._lengths_c is None or self._lengths_c[0] != lengths:
            self._lengths_c = (lengths, (C.c_int * len(lengths))(*lengths))
        return self._lengths_c[1]

    def close(self):
        """Writes every generator's offset back: its offset at the start plus what the draws consumed."""
        if self.draws:
            for g, s, inc in zip(self.generators, self.start, self.incs):
                g.set_offset(s + self.draws * int(inc))
        self.draws = 0
