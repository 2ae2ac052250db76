"""Seeded per-sample sampling: the ``seeds=`` argument of the samplers.

With ``seeds`` (one int64 in [0, 2^63) per sample) every random draw of a sampler run comes from the counter-based generator
``dsb_seeded_normal`` (include/diffsbdd_b200.h) instead of torch's global generator: Philox4x32-10 keyed by the sample's
own seed, with a counter made of the draw id, the role (ligand rows, pocket rows, the joint model's shared coordinate
noise, one row per graph) and the row's index within its own graph.  A sample's noise is then the same whatever batch,
batch position or GPU count drew it, and in deterministic mode (``EGNNDynamics.deterministic``) so is the sample.

Draw id (int64): ``stage << 40 | s << 20 | u << 4 | purpose``.  ``stage`` is where in the run the draw happens, ``s`` the
reverse step, ``u`` the resampling round (RePaint: the resampling index of the conditional model, the number of jumps back
so far of the joint model) and ``purpose`` which of a step's draws it is.  The captured CUDA-graph steps compute it on the
device from their step counter, so one capture serves every step and every set of seeds.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import _native

STAGE_PRIOR, STAGE_LOOP, STAGE_FINAL, STAGE_PARTIAL, STAGE_SIZE = 0, 1, 2, 3, 4
PURPOSE_REVERSE, PURPOSE_KNOWN, PURPOSE_RENOISE = 0, 1, 2
_S_BITS, _U_BITS = 20, 16


def draw_id(stage: int, s: int = 0, u: int = 0, purpose: int = 0) -> int:
    if not (0 <= s < (1 << _S_BITS) and 0 <= u < (1 << _U_BITS) and 0 <= purpose < 16 and 0 <= stage < 16):
        raise ValueError(f'draw id out of range: stage={stage} s={s} u={u} purpose={purpose}')
    return (stage << 40) | (s << 20) | (u << 4) | purpose


def check_schedule(timesteps: int, rounds: int = 1) -> None:
    """Raises before a seeded run starts if its steps or resampling rounds (RePaint resamplings, joint-model jump blocks)
    do not fit the draw-id fields: 20 bits for s, 16 for u.  Past them two different draws would reuse one noise."""
    if not (0 < timesteps <= (1 << _S_BITS) and 0 < rounds <= (1 << _U_BITS)):
        raise ValueError(f'seeded sampling supports at most {1 << _S_BITS} steps and {1 << _U_BITS} resampling rounds '
                         f'per run, got {timesteps} steps and {rounds} rounds')


def as_seeds(seeds, n_samples: int, device) -> Optional[torch.Tensor]:
    """Validated int64 seeds on ``device`` (None stays None).  Accepts a sequence of ints, a numpy array or an integer
    tensor on any device; one value per sample, each in [0, 2^63).  Seeded sampling needs the CUDA generator: a CPU run
    raises."""
    if seeds is None:
        return None
    if torch.device(device).type != 'cuda':
        raise RuntimeError('seeds= needs a CUDA device: the seeded generator is a CUDA kernel')
    return host_seeds(seeds, n_samples).to(device)


def host_seeds(seeds, n_samples: int) -> torch.Tensor:
    """The validation of ``as_seeds``: a CPU int64 tensor of ``n_samples`` values in [0, 2^63), or an exception."""
    if isinstance(seeds, torch.Tensor):
        if seeds.dtype.is_floating_point or seeds.dtype.is_complex or seeds.dtype == torch.bool:
            raise TypeError(f'seeds must be an integer tensor, got {seeds.dtype}')
        host = seeds.detach().cpu().to(torch.int64)        # an unsigned value >= 2^63 wraps negative and fails below
    else:
        arr = np.asarray(seeds)
        if arr.dtype == object or not (np.issubdtype(arr.dtype, np.integer) or arr.size == 0):
            raise TypeError(f'seeds must be integers, got {arr.dtype}')
        if np.issubdtype(arr.dtype, np.unsignedinteger) and arr.size and int(arr.max()) >= 1 << 63:
            raise ValueError('seeds must lie in [0, 2^63)')
        host = torch.from_numpy(arr.astype(np.int64))
    if host.dim() != 1 or host.numel() != n_samples:
        raise ValueError(f'seeds must hold one value per sample: {n_samples} expected, got shape {tuple(host.shape)}')
    if host.numel() and int(host.min()) < 0:
        raise ValueError('seeds must lie in [0, 2^63)')
    return host.contiguous()


def fill(out: torch.Tensor, role: int, seeds: torch.Tensor, draw: torch.Tensor, lig_mask: Optional[torch.Tensor],
         pocket_mask: Optional[torch.Tensor], kind: int = _native.RNG_NORMAL) -> torch.Tensor:
    """One dsb_seeded_normal launch into the contiguous fp32 ``out`` [rows, cols] on the current stream.  ``draw`` is a
    device int64 tensor whose first element is the draw id (read when the kernel runs)."""
    import ctypes as C
    assert out.is_contiguous() and out.dtype == torch.float32 and draw.dtype == torch.int64
    nl = 0 if lig_mask is None else len(lig_mask)
    npk = 0 if pocket_mask is None else len(pocket_mask)
    ptr = lambda x: None if x is None else x.data_ptr()
    _native.check(_native.load().dsb_seeded_normal(
        ptr(out), out.shape[1] if out.dim() == 2 else 1, role, kind, ptr(seeds), ptr(draw), ptr(lig_mask), ptr(pocket_mask),
        nl, npk, len(seeds), C.c_void_p(torch.cuda.current_stream(out.device).cuda_stream)))
    return out


class SeededDraws:
    """The generator state of one seeded sampler call: seeds, masks and the draw id the next draws use (``at``)."""

    def __init__(self, seeds: torch.Tensor, lig_mask: torch.Tensor, pocket_mask: torch.Tensor):
        self.seeds, self.lig_mask, self.pocket_mask = seeds, lig_mask, pocket_mask
        self.draw = draw_id(STAGE_PRIOR)

    def at(self, stage: int, s: int = 0, u: int = 0, purpose: int = 0) -> 'SeededDraws':
        self.draw = draw_id(stage, s, u, purpose)
        return self

    def normal(self, role: int, cols: int) -> torch.Tensor:
        rows = {_native.RNG_LIGAND: len(self.lig_mask), _native.RNG_POCKET: len(self.pocket_mask),
                _native.RNG_JOINT_X: len(self.lig_mask) + len(self.pocket_mask), _native.RNG_GRAPH: len(self.seeds)}[role]
        out = torch.empty((rows, cols), device=self.seeds.device)
        d = torch.full((1,), self.draw, dtype=torch.int64, device=self.seeds.device)
        return fill(out, role, self.seeds, d, self.lig_mask, self.pocket_mask)


def graph_draw_ids(step: torch.Tensor, u: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """Device-side draw ids of one captured reverse step: out[p] = draw_id(STAGE_LOOP, step, u, p) for p = 0..len(out)-1."""
    base = (STAGE_LOOP << 40) + step.clamp(min=0) * (1 << _S_BITS) + u * (1 << 4)
    torch.add(base, torch.arange(out.numel(), device=out.device, dtype=torch.int64), out=out)
    return out


def size_prior(prob: torch.Tensor, n_pocket: torch.Tensor, seeds: torch.Tensor) -> torch.Tensor:
    """Ligand sizes ~ p(n_lig | n_pocket) by inverse CDF, one seeded uniform per sample (stage STAGE_SIZE, role GRAPH):
    n = the smallest i with u <= cdf_j[i], cdf_j = cumsum(prob[:, j]) / sum(prob[:, j]) in float64, j = the pocket size."""
    device = seeds.device
    u = torch.empty((len(seeds), 1), device=device)
    fill(u, _native.RNG_GRAPH, seeds, torch.full((1,), draw_id(STAGE_SIZE), dtype=torch.int64, device=device), None, None,
         _native.RNG_UNIFORM)
    return inverse_cdf(prob.to(device), n_pocket.to(device), u.view(-1))


def inverse_cdf(prob: torch.Tensor, n_pocket: torch.Tensor, u: torch.Tensor) -> torch.Tensor:
    cdf = torch.cumsum(prob.double(), dim=0)[:, n_pocket.long()].T          # [n_samples, n_lig_bins]
    cdf = cdf / cdf[:, -1:]
    idx = torch.searchsorted(cdf.contiguous(), u.double().view(-1, 1)).view(-1)
    return idx.clamp(max=prob.shape[0] - 1)
