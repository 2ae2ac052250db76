"""Multi-GPU sampling: the path shards by pocket (SURVEY.md §8(e)).

Graphs are independent (edges never cross graphs — dynamics.py:115, :170-172) and the DDPM loop carries state per graph
only, so a batch of pockets is split contiguously across ranks; every rank runs the full reverse loop on its own shard with
seed ``base_seed + rank`` and NO collective inside the loop.  The only exchange is one gather of the generated ligands at the
end (``[N_L_rank, 3+atom_nf]`` fp32 + the ligand sizes).  One process per GPU (torchrun); NCCL on GPUs, gloo in the CPU tests.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import torch
import torch.distributed as dist

from .en_diffusion import check_sampler


def shard_bounds(n_items: int, world_size: int, rank: int) -> Tuple[int, int]:
    """Contiguous split of ``n_items`` pockets; the first ``n_items % world_size`` ranks get one extra."""
    base, extra = divmod(n_items, world_size)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_pocket(pocket: Dict[str, torch.Tensor], lo: int, hi: int) -> Dict[str, torch.Tensor]:
    """Sub-batch [lo, hi) of a reference ``pocket`` dict {'x','one_hot','size','mask'} with graph ids renumbered from 0."""
    sizes = pocket['size']
    starts = torch.cumsum(sizes, 0) - sizes
    a = int(starts[lo]) if lo < len(sizes) else int(sizes.sum())
    b = int(starts[hi - 1] + sizes[hi - 1]) if hi > lo else a
    return {'x': pocket['x'][a:b], 'one_hot': pocket['one_hot'][a:b], 'size': sizes[lo:hi], 'mask': pocket['mask'][a:b] - lo}


@torch.no_grad()
def shard_seeds(seeds, lo: int, hi: int) -> torch.Tensor:
    """This rank's slice [lo, hi) of the whole job's per-sample seeds, as an int64 tensor."""
    seeds = seeds if isinstance(seeds, torch.Tensor) else torch.as_tensor(seeds, dtype=torch.int64)
    return seeds[lo:hi]


@torch.no_grad()
def sample_given_pocket_sharded(ddpm, pocket: Dict[str, torch.Tensor], num_nodes_lig: torch.Tensor, base_seed: int = 0,
                                timesteps=None, group=None, seeds=None, sampler='ddpm', eta=0.0):
    """Runs ``ddpm.sample_given_pocket`` on this rank's shard of the pockets and gathers the ligands of all ranks.

    ``pocket``/``num_nodes_lig`` describe the WHOLE job on every rank (device tensors of this rank).  Returns
    ``(xh_lig_all, lig_sizes_all)`` — identical on every rank, ordered by global pocket index — plus this rank's own
    ``(xh_lig, xh_pocket, lig_mask, pocket_mask)`` tuple.

    ``seeds`` (one int64 per pocket of the whole job): rank r samples its pockets with ``seeds[lo:hi]`` and ``base_seed`` is
    ignored, so in deterministic mode the gathered ligands are the same for any number of ranks.  Without ``seeds`` every
    rank draws from torch's generator seeded with ``base_seed + rank``.  ``sampler`` / ``eta``: as
    ``ConditionalDDPM.sample_given_pocket``.
    """
    check_sampler(sampler, eta)
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    n = len(pocket['size'])
    lo, hi = shard_bounds(n, world, rank)
    dev = pocket['x'].device
    gen_state = torch.random.get_rng_state()
    if seeds is not None:
        if len(seeds) != n:
            raise ValueError(f'seeds must hold one value per pocket of the whole job: {n} expected, got {len(seeds)}')
        local_seeds = shard_seeds(seeds, lo, hi)
    else:
        local_seeds = None
        torch.manual_seed(base_seed + rank)
        if dev.type == 'cuda':
            torch.cuda.manual_seed(base_seed + rank)
    if hi > lo:
        extra = {} if local_seeds is None else {'seeds': local_seeds}
        if sampler != 'ddpm':
            extra.update(sampler=sampler, eta=eta)
        local = ddpm.sample_given_pocket(shard_pocket(pocket, lo, hi), num_nodes_lig[lo:hi], timesteps=timesteps, **extra)
    else:
        width = ddpm.n_dims + ddpm.atom_nf
        local = (torch.zeros((0, width), device=dev), torch.zeros((0, ddpm.n_dims + ddpm.residue_nf), device=dev),
                 torch.zeros(0, dtype=torch.int64, device=dev), torch.zeros(0, dtype=torch.int64, device=dev))
    torch.random.set_rng_state(gen_state)
    xh_lig = local[0].contiguous().float()
    sizes_all = num_nodes_lig.to(dev)
    if world == 1:
        return xh_lig, sizes_all, local
    # fixed-size all_gather: every rank pads its ligand block to the largest shard
    counts = [int(sizes_all[slice(*shard_bounds(n, world, r))].sum()) for r in range(world)]
    width = xh_lig.shape[1]
    pad = torch.zeros((max(counts), width), dtype=torch.float32, device=dev)
    pad[:xh_lig.shape[0]] = xh_lig
    bufs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(bufs, pad, group=group)
    xh_all = torch.cat([b[:c] for b, c in zip(bufs, counts)], dim=0)
    return xh_all, sizes_all, local
