"""Seeded synthetic weights and pocket+ligand batches (SURVEY.md §8(d)).

No checkpoint and no dataset is reachable offline, so every benchmark and parity test uses:

* weights that are a pure function of ``(state-dict key, shape, seed)`` — independent of module
  construction order, so the same tensors can be loaded into the unmodified reference modules
  (``load_state_dict``) and into this package's ``EGNNDynamics``;
* pocket geometry: points uniform in a ball at a given number density (0.045 A^-3 full-atom,
  0.007 A^-3 C-alpha), centred; ligand start state as in conditional_model.py:502-508.

The state-dict layout follows the reference modules (dynamics.py:27-53, egnn_new.py:15-29,
:78-92, :212-222); see SURVEY.md §8(b) "state dict".
"""
from __future__ import annotations

import hashlib
import math
from typing import Dict, List, Tuple

import torch

from .config import DynamicsConfig


def state_dict_spec(cfg: DynamicsConfig) -> List[Tuple[str, Tuple[int, ...], int]]:
    """(key, shape, fan_in) for every parameter the reference ``EGNNDynamics`` owns."""
    A, R, J, H = cfg.atom_nf, cfg.residue_nf, cfg.joint_nf, cfg.hidden_nf
    Din = J + (1 if cfg.condition_time else 0)
    F = cfg.edge_feat_nf
    spec: List[Tuple[str, Tuple[int, ...], int]] = []

    def lin(prefix, out_f, in_f, bias=True):
        spec.append((prefix + '.weight', (out_f, in_f), in_f))
        if bias:
            spec.append((prefix + '.bias', (out_f,), in_f))

    lin('atom_encoder.0', 2 * A, A)
    lin('atom_encoder.2', J, 2 * A)
    lin('atom_decoder.0', 2 * A, J)
    lin('atom_decoder.2', A, 2 * A)
    lin('residue_encoder.0', 2 * R, R)
    lin('residue_encoder.2', J, 2 * R)
    lin('residue_decoder.0', 2 * R, J)
    lin('residue_decoder.2', R, 2 * R)
    if cfg.edge_embedding_dim:
        spec.append(('edge_embedding.weight', (3, cfg.edge_embedding_dim), 1))
    lin('egnn.embedding', H, Din)
    lin('egnn.embedding_out', Din, H)
    for k in range(cfg.n_layers):
        b = f'egnn.e_block_{k}'
        for s in range(cfg.inv_sublayers):
            g = f'{b}.gcl_{s}'
            lin(g + '.edge_mlp.0', H, 2 * H + F)
            lin(g + '.edge_mlp.2', H, H)
            lin(g + '.node_mlp.0', H, 2 * H)
            lin(g + '.node_mlp.2', H, H)
            if cfg.attention:
                lin(g + '.att_mlp.0', 1, H)
        q = f'{b}.gcl_equiv'
        lin(q + '.coord_mlp.0', H, 2 * H + F)
        lin(q + '.coord_mlp.2', H, H)
        lin(q + '.coord_mlp.4', 1, H, bias=False)
        if not cfg.reflection_equivariant:
            lin(q + '.cross_product_mlp.0', H, 2 * H + F)
            lin(q + '.cross_product_mlp.2', H, H)
            # '.cross_product_mlp.4.weight' aliases coord_mlp.4.weight (egnn_new.py:78,85,91)
    return spec


def _key_seed(key: str, seed: int) -> int:
    d = hashlib.sha256(f'{seed}:{key}'.encode()).digest()
    return int.from_bytes(d[:7], 'little')


def synthetic_state_dict(cfg: DynamicsConfig, seed: int = 0,
                         coord_out_scale: float = 0.05) -> Dict[str, torch.Tensor]:
    """Weights ~ U(-1/sqrt(fan_in), 1/sqrt(fan_in)) per key (the nn.Linear default family).

    The bias-free last coordinate layer (reference init: xavier gain 0.001, egnn_new.py:79) is
    drawn from U(-coord_out_scale, coord_out_scale) instead (about 300x the reference bound) so the coordinate outputs are O(0.1-1) rather
    than O(1e-4) — otherwise coordinate parity would be vacuous (SURVEY.md §8(c)).
    """
    sd: Dict[str, torch.Tensor] = {}
    for key, shape, fan_in in state_dict_spec(cfg):
        g = torch.Generator(device='cpu')
        g.manual_seed(_key_seed(key, seed))
        bound = 1.0 / math.sqrt(max(fan_in, 1))
        if key.endswith('coord_mlp.4.weight'):
            bound = coord_out_scale
        if key == 'edge_embedding.weight':
            bound = 1.0
        t = (torch.rand(shape, generator=g, dtype=torch.float64) * 2.0 - 1.0) * bound
        sd[key] = t.to(torch.float32)
    if not cfg.reflection_equivariant:
        for k in range(cfg.n_layers):
            q = f'egnn.e_block_{k}.gcl_equiv'
            sd[q + '.cross_product_mlp.4.weight'] = sd[q + '.coord_mlp.4.weight']
    return sd


def state_dict_checksum(sd: Dict[str, torch.Tensor]) -> float:
    """Order-independent fingerprint used by the golden fixtures to pin the weight recipe."""
    tot = 0.0
    for k in sorted(sd):
        v = sd[k].double()
        idx = torch.arange(1, v.numel() + 1, dtype=torch.float64)
        tot += float((v.flatten() * torch.sin(idx)).sum())
    return tot


def _ball_points(n: int, density: float, g: torch.Generator) -> torch.Tensor:
    radius = (n / density / (4.0 * math.pi / 3.0)) ** (1.0 / 3.0)
    pts = torch.empty((0, 3), dtype=torch.float64)
    while pts.shape[0] < n:
        c = (torch.rand((4 * n + 16, 3), generator=g, dtype=torch.float64) * 2 - 1) * radius
        c = c[(c ** 2).sum(1) <= radius ** 2]
        pts = torch.cat([pts, c])
    pts = pts[:n]
    return pts - pts.mean(0, keepdim=True)


def synthetic_pocket(cfg: DynamicsConfig, n_pocket, seed: int = 0, density: float = 0.045,
                     spread: float = 0.0) -> Dict[str, torch.Tensor]:
    """Reference ``pocket`` dict {'x','one_hot','size','mask'} (lightning_modules.py:745-750),
    un-normalised (Angstrom coordinates, 0/1 one-hot). ``n_pocket`` int list or int per graph.
    ``spread`` displaces whole pockets from the origin (tests translation handling)."""
    g = torch.Generator(device='cpu')
    g.manual_seed(_key_seed('pocket', seed))
    sizes = list(n_pocket)
    xs, hs, masks = [], [], []
    for b, n in enumerate(sizes):
        x = _ball_points(n, density, g)
        if spread:
            x = x + (torch.rand((1, 3), generator=g, dtype=torch.float64) * 2 - 1) * spread
        xs.append(x)
        types = torch.randint(0, cfg.residue_nf, (n,), generator=g)
        hs.append(torch.nn.functional.one_hot(types, cfg.residue_nf))
        masks.append(torch.full((n,), b, dtype=torch.int64))
    return {
        'x': torch.cat(xs).to(torch.float32),
        'one_hot': torch.cat(hs).to(torch.float32),
        'size': torch.tensor(sizes, dtype=torch.int64),
        'mask': torch.cat(masks),
    }


def synthetic_complex_batch(cfg: DynamicsConfig, n_lig, n_pocket, seed: int = 0, density: float = 0.045,
                            lig_sigma: float = 1.5) -> Dict[str, torch.Tensor]:
    """A batch dict with the keys of the reference datasets (lightning_modules.py:217-234) for likelihood evaluation:
    ``synthetic_pocket`` pockets with ligands ~ N(pocket COM, lig_sigma^2) and random atom types."""
    p = synthetic_pocket(cfg, n_pocket, seed=seed, density=density)
    g = torch.Generator(device='cpu')
    g.manual_seed(_key_seed('ligand', seed))
    sizes = torch.tensor(list(n_lig), dtype=torch.int64)
    mask = torch.repeat_interleave(torch.arange(len(sizes)), sizes)
    com = torch.zeros((len(sizes), 3)).index_add_(0, p['mask'], p['x']) / p['size'].clamp(min=1).unsqueeze(1).float()
    x = com[mask] + lig_sigma * torch.randn((len(mask), 3), generator=g)
    types = torch.randint(0, cfg.atom_nf, (len(mask),), generator=g)
    return {'lig_coords': x, 'lig_one_hot': torch.nn.functional.one_hot(types, cfg.atom_nf).float(),
            'num_lig_atoms': sizes, 'lig_mask': mask, 'pocket_coords': p['x'], 'pocket_one_hot': p['one_hot'],
            'num_pocket_nodes': p['size'], 'pocket_mask': p['mask']}


def synthetic_denoiser_inputs(cfg: DynamicsConfig, n_lig, n_pocket, seed: int = 0,
                              density: float = 0.045, t_value=None,
                              norm_values=(1.0, 4.0), lig_sigma: float = 1.0):
    """One ``EGNNDynamics.forward`` argument tuple on CPU (reference dynamics.py:87).

    Pocket: normalised as en_diffusion.py:880-895; ligand: z ~ N(pocket COM, sigma) with the ligand
    COM removed from both (conditional_model.py:502-508, :151-158). ``t_value`` None draws one
    t in (0,1) per graph.
    """
    n_lig, n_pocket = list(n_lig), list(n_pocket)
    assert len(n_lig) == len(n_pocket)
    B = len(n_lig)
    pocket = synthetic_pocket(cfg, n_pocket, seed, density)
    g = torch.Generator(device='cpu')
    g.manual_seed(_key_seed('ligand', seed))
    mask_res = pocket['mask']
    mask_at = torch.repeat_interleave(torch.arange(B), torch.tensor(n_lig))
    x_p = pocket['x'].double() / norm_values[0]
    h_p = pocket['one_hot'].double() / norm_values[1]
    com = torch.zeros((B, 3), dtype=torch.float64).index_add_(0, mask_res, x_p)
    com = com / torch.tensor(n_pocket, dtype=torch.float64)[:, None]
    z = torch.randn((len(mask_at), 3 + cfg.atom_nf), generator=g, dtype=torch.float64) * lig_sigma
    z[:, :3] += com[mask_at]
    lig_mean = torch.zeros((B, 3), dtype=torch.float64).index_add_(0, mask_at, z[:, :3])
    lig_mean = lig_mean / torch.tensor(n_lig, dtype=torch.float64)[:, None]
    z[:, :3] -= lig_mean[mask_at]
    x_p = x_p - lig_mean[mask_res]
    xh_res = torch.cat([x_p, h_p], 1)
    if t_value is None:
        t = torch.rand((B, 1), generator=g, dtype=torch.float64)
    else:
        t = torch.full((B, 1), float(t_value), dtype=torch.float64)
    return (z.to(torch.float32), xh_res.to(torch.float32), t.to(torch.float32),
            mask_at.to(torch.int64), mask_res.to(torch.int64))


def min_cutoff_margin(cfg: DynamicsConfig, xh_atoms, xh_residues, mask_atoms, mask_residues) -> float:
    """Smallest | d_ij - cutoff | over same-graph pairs: fixtures must keep this well above
    fp32 rounding so the edge set is implementation-independent (SURVEY.md §7 'Edge set numerics')."""
    xa, xr = xh_atoms[:, :3].double(), xh_residues[:, :3].double()
    best = float('inf')
    for (xa_, xb_, ma, mb, c) in ((xa, xa, mask_atoms, mask_atoms, cfg.edge_cutoff_ligand),
                                  (xr, xr, mask_residues, mask_residues, cfg.edge_cutoff_pocket),
                                  (xa, xr, mask_atoms, mask_residues, cfg.edge_cutoff_interaction)):
        if c is None or len(xa_) == 0 or len(xb_) == 0:
            continue
        d = torch.cdist(xa_, xb_)
        same = ma[:, None] == mb[None, :]
        if same.any():
            best = min(best, float((d[same] - c).abs().min()))
    return best
