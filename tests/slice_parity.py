"""TEST INFRASTRUCTURE ONLY -- the sliced parity rule: every slice of a model output within the 16-bit oracle's own error.

A whole-output relative L2 dilutes a local error by the square root of the fraction of the output it touches: a frame sent
to the wrong modulation row, a caption token dropped from one sample's cross-attention or one row tile of a GEMM left
unwritten moves the whole-output error by a few per cent of the oracle's own 16-bit error.  This rule cuts the output into
slices, one per (sample, frame, 128-row token tile, 128-column channel tile), and asks of every slice s

    ||ours - r32||_s  <=  K * ||r16 - r32||_s  +  FLOOR * ||r16 - r32|| / sqrt(#slices)

where r16 is the oracle (or reference) in the 16-bit dtype and r32 the same in fp32.  The second term is a floor of a
quarter of the RMS per-slice share of the oracle's own error, so that slices where the output is nearly zero do not fail
on noise.  ``load`` = left side / right side; a slice passes when its load is at most 1.  An output narrower than 128
channels (a latent) keeps all its channels in one slice and takes token tiles of 128 * ceil(128 / C) rows, so that its
slices hold as many elements as a 128 x 128 tile: on 128 elements a ratio of two norms scatters by tens of per cent.

Axes name the dimensions of the output: ``b`` sample, ``t`` frame, ``n`` token (several ``n`` dimensions, e.g. the rows
and columns of a latent, flatten row-major into one token index), ``c`` channel.  A missing letter is an axis of extent 1.
Golden files of large cases keep a seeded sample of the output elements and their flat index; ``idx`` / ``shape`` take
that form, and the sampled elements are grouped by (sample, frame) only.
"""
import math
from dataclasses import dataclass
from typing import Optional, Sequence

import torch

TILE = 128
K = 1.25
FLOOR = 0.25
OLD_K = 1.25  # the whole-output gate: ||ours - r32|| <= OLD_K * ||r16 - r32|| + 1e-4 ||r32||


@dataclass
class SliceReport:
    name: str
    grid: tuple  # slices per axis: (samples, frames, token tiles, channel tiles)
    tile: tuple  # (token rows, channels) per slice
    loads: torch.Tensor  # [grid] err_s / bound_s
    ratios: torch.Tensor  # [grid] err_s / ref_s
    worst_at: tuple  # (sample, frame, first token, first channel) of the worst slice
    worst_err: float
    worst_ref: float
    floor: float
    whole_ratio: float  # ||ours - r32|| / ||r16 - r32||
    old_gate_ok: bool

    @property
    def worst(self) -> float:
        return float(self.loads.max())

    @property
    def ok(self) -> bool:
        return self.worst <= 1.0

    def describe(self) -> str:
        q = torch.tensor([0.5, 0.9, 0.99, 1.0], dtype=torch.float64)
        lq = torch.quantile(self.loads.flatten(), q).tolist()
        rq = torch.quantile(self.ratios.flatten().clamp(max=1e6), q).tolist()
        b, t, n, c = self.worst_at
        return (f"[slices] {self.name}: {self.loads.numel()} slices {self.grid} of {self.tile[0]} tokens x {self.tile[1]} channels; "
                f"worst load {self.worst:.3f} at sample {b} frame {t} tokens {n}.. channels {c}.. "
                f"(err {self.worst_err:.3e}, own 16-bit err {self.worst_ref:.3e}, floor {self.floor:.3e}); "
                f"load p50/p90/p99/max {lq[0]:.3f}/{lq[1]:.3f}/{lq[2]:.3f}/{lq[3]:.3f}; "
                f"err/own p50/p90/p99/max {rq[0]:.3f}/{rq[1]:.3f}/{rq[2]:.3f}/{rq[3]:.3f}; "
                f"whole-output err/own {self.whole_ratio:.3f} (old {OLD_K}x gate {'passes' if self.old_gate_ok else 'fails'})")


def _perm(axes: str, ndim: int):
    if len(axes) != ndim or set(axes) - set("btnc"):
        raise ValueError(f"axes {axes!r} must name each of the {ndim} dimensions with one of b, t, n, c")
    return [i for a in "btnc" for i, x in enumerate(axes) if x == a]


def _extents(axes: str, shape: Sequence[int]):
    """(B, T, N, C): the products of the extents named by each letter."""
    return tuple(math.prod(s for a, s in zip(axes, shape) if a == x) for x in "btnc")


def _canon(t: torch.Tensor, axes: str) -> torch.Tensor:
    """t as float64 [B, T, N, C]."""
    return t.double().permute(_perm(axes, t.dim())).reshape(_extents(axes, t.shape))


def _tile_sq(d: torch.Tensor, tn: int, tc: int) -> torch.Tensor:
    """Per-slice sums of squares of d [B, T, N, C]: [B, T, ceil(N/tn), ceil(C/tc)]."""
    B, T, N, C = d.shape
    nt, ct = -(-N // tn), -(-C // tc)
    d = torch.nn.functional.pad(d * d, (0, ct * tc - C, 0, nt * tn - N))
    return d.view(B, T, nt, tn, ct, tc).sum(dim=(3, 5))


def sliced_parity(name: str, ours, r16, r32, axes: str, idx: Optional[torch.Tensor] = None,
                  shape: Optional[Sequence[int]] = None, k: float = K, floor: float = FLOOR) -> SliceReport:
    """The rule on full outputs of the shape the axes describe, or, with idx and shape, on the elements idx (flat indices
    into an output of that shape) of it: ours / r16 / r32 then hold those elements in the order of idx."""
    if idx is None:
        o, a, r = (_canon(x, axes) for x in (ours, r16, r32))
        assert o.shape == a.shape == r.shape, (ours.shape, r16.shape, r32.shape)
        B, T, N, C = o.shape
        # a narrow output (a latent) keeps its channels together and takes taller token tiles, so that every slice
        # holds about TILE x TILE elements: a norm over 128 elements scatters by tens of per cent on its own
        tn, tc = (TILE, TILE) if C >= TILE else (TILE * -(-TILE // C), C)
        err2, ref2 = _tile_sq(o - r, tn, tc), _tile_sq(a - r, tn, tc)
        tot_r, tot_e = r.norm().item(), (o - r).norm().item()
    else:
        shape = tuple(shape)
        o, a, r = (x.double().flatten() for x in (ours, r16, r32))
        assert o.shape == a.shape == r.shape == idx.shape, (ours.shape, r16.shape, r32.shape, idx.shape)
        B, T, N, C = _extents(axes, shape)
        coord = torch.stack(torch.unravel_index(idx.long(), shape))  # [ndim, n]
        bt = torch.zeros_like(idx, dtype=torch.long)
        for letter in "bt":  # row-major over the b dimensions, then the t dimensions
            for i, x in enumerate(axes):
                if x == letter:
                    bt = bt * shape[i] + coord[i]
        tn, tc = N, C
        err2 = torch.zeros(B * T, dtype=torch.float64).index_add_(0, bt, (o - r) ** 2).view(B, T, 1, 1)
        ref2 = torch.zeros(B * T, dtype=torch.float64).index_add_(0, bt, (a - r) ** 2).view(B, T, 1, 1)
        tot_r, tot_e = r.norm().item(), (o - r).norm().item()
    err, ref = err2.sqrt(), ref2.sqrt()
    tot_ref = ref2.sum().sqrt().item()
    fl = floor * tot_ref / math.sqrt(err.numel())
    loads = err / (k * ref + fl)
    ratios = err / ref.clamp_min(1e-300)
    w = int(loads.flatten().argmax())
    b, t, i, j = torch.unravel_index(torch.tensor(w), loads.shape)
    return SliceReport(name=name, grid=tuple(loads.shape), tile=(tn, tc), loads=loads, ratios=ratios,
                       worst_at=(int(b), int(t), int(i) * tn, int(j) * tc), worst_err=err.flatten()[w].item(),
                       worst_ref=ref.flatten()[w].item(), floor=fl, whole_ratio=tot_e / max(tot_ref, 1e-300),
                       old_gate_ok=tot_e <= OLD_K * tot_ref + 1e-4 * tot_r)


def assert_sliced_parity(name: str, ours, r16, r32, axes: str, **kw) -> SliceReport:
    """sliced_parity, printed, and asserted."""
    rep = sliced_parity(name, ours, r16, r32, axes, **kw)
    print(rep.describe())
    assert rep.ok, (f"{name}: slice at sample {rep.worst_at[0]} frame {rep.worst_at[1]} tokens {rep.worst_at[2]}.. "
                    f"channels {rep.worst_at[3]}.. is {rep.worst:.3f}x its bound")
    return rep
