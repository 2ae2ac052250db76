"""TEST INFRASTRUCTURE ONLY — CPU oracle for the denoiser hot path.

A functional, state-dict-driven restatement of what ``EGNNDynamics.forward`` computes in the
reference (dynamics.py:87-167 -> egnn_new.py:225-244 -> :163-184 -> :60-66, :124-132). It exists so
that the parity tests, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline leg have a checker
that travels with the repository (the reference checkout is not needed to run them). The product path
(``diffsbdd_b200``) never imports this module.

Parity pinning: the reference ships no golden vectors (SURVEY.md §8(c)); this oracle is pinned
instead against stored outputs of the unmodified reference
(``tests/golden/*.npz`` produced by ``tests/golden/make_golden.py`` through ``oracle/ref_shim.py``).

The op sequence deliberately follows the reference (materialised ``[h_i | h_j | e_ij]`` concatenation,
whole-batch ``cdist`` adjacency) so that (i) fp32 results agree with the reference to the last bit
or two on CPU and (ii) timing it is a fair stand-in for "the reference's own PyTorch CPU path".
Works in float32 (default) or float64 (a higher-precision truth for tolerance studies).
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import math

import torch
import torch.nn.functional as F


def _linear(sd, prefix, x):
    w = sd[prefix + '.weight']
    b = sd.get(prefix + '.bias')
    return F.linear(x, w, b)


def _mlp2(sd, prefix, x):
    """Linear -> SiLU -> Linear (dynamics.py:27-49: encoders/decoders)."""
    return _linear(sd, prefix + '.2', F.silu(_linear(sd, prefix + '.0', x)))


def segment_sum(data, segment_ids, num_segments, normalization_factor, aggregation_method):
    """egnn_new.py:319-335 (``unsorted_segment_sum``): zero-init, scatter-add along dim 0, then
    '/normalization_factor' for 'sum' or '/count (0 -> 1)' for 'mean'."""
    out = torch.zeros((num_segments, data.shape[1]), dtype=data.dtype, device=data.device)
    idx = segment_ids.unsqueeze(-1).expand(-1, data.shape[1])
    out.scatter_add_(0, idx, data)
    if aggregation_method == 'sum':
        out = out / normalization_factor
    if aggregation_method == 'mean':
        cnt = torch.zeros_like(out)
        cnt.scatter_add_(0, idx, torch.ones_like(data))
        cnt[cnt == 0] = 1
        out = out / cnt
    return out


def radial_and_direction(x, row, col, norm_constant):
    """egnn_new.py:296-302 (``coord2diff``): d^2 and (x_i-x_j)/(sqrt(d^2+1e-8)+norm_constant)."""
    diff = x[row] - x[col]
    radial = torch.sum(diff ** 2, 1).unsqueeze(1)
    norm = torch.sqrt(radial + 1e-8)
    return radial, diff / (norm + norm_constant)


def cross_direction(x, row, col, batch_mask, norm_constant):
    """egnn_new.py:305-316 (``coord2cross``): normalised cross product about the per-graph centroid
    of ALL nodes (ligand+pocket) at the current coordinates."""
    n_graphs = int(batch_mask.max()) + 1
    mean = segment_sum(x, batch_mask, n_graphs, None, 'mean')
    c = torch.cross(x[row] - mean[batch_mask[row]], x[col] - mean[batch_mask[col]], dim=1)
    nrm = torch.linalg.norm(c, dim=1, keepdim=True)
    return c / (nrm + norm_constant)


def build_edges(cfg, mask_lig, mask_pocket, x_lig, x_pocket):
    """dynamics.py:169-187 (``get_edges``): same-graph AND (cdist <= cutoff) per block type, ligand
    block / cross block / pocket block assembled [[LL, LP], [LP^T, PP]], ``where`` -> row-major [2,E]."""
    a_ll = mask_lig[:, None] == mask_lig[None, :]
    a_pp = mask_pocket[:, None] == mask_pocket[None, :]
    a_lp = mask_lig[:, None] == mask_pocket[None, :]
    if cfg.edge_cutoff_ligand is not None:
        a_ll = a_ll & (torch.cdist(x_lig, x_lig) <= cfg.edge_cutoff_ligand)
    if cfg.edge_cutoff_pocket is not None:
        a_pp = a_pp & (torch.cdist(x_pocket, x_pocket) <= cfg.edge_cutoff_pocket)
    if cfg.edge_cutoff_interaction is not None:
        a_lp = a_lp & (torch.cdist(x_lig, x_pocket) <= cfg.edge_cutoff_interaction)
    top = torch.cat((a_ll, a_lp), dim=1)
    bottom = torch.cat((a_lp.T, a_pp), dim=1)
    row, col = torch.where(torch.cat((top, bottom), dim=0))
    return torch.stack((row, col), dim=0)


def gcl(sd, prefix, cfg, h, row, col, edge_attr):
    """egnn_new.py:60-66 / :31-58: edge MLP (+attention gate), receiver-side segment sum, node MLP
    with residual."""
    m = torch.cat([h[row], h[col], edge_attr], dim=1)
    m = F.silu(_linear(sd, prefix + '.edge_mlp.2', F.silu(_linear(sd, prefix + '.edge_mlp.0', m))))
    if cfg.attention:
        m = m * torch.sigmoid(_linear(sd, prefix + '.att_mlp.0', m))
    agg = segment_sum(m, row, h.shape[0], cfg.normalization_factor, cfg.aggregation_method)
    z = torch.cat([h, agg], dim=1)
    return h + _linear(sd, prefix + '.node_mlp.2', F.silu(_linear(sd, prefix + '.node_mlp.0', z)))


def _scalar_mlp3(sd, prefix, z):
    y = F.silu(_linear(sd, prefix + '.0', z))
    y = F.silu(_linear(sd, prefix + '.2', y))
    return _linear(sd, prefix + '.4', y)


def equivariant_update(sd, prefix, cfg, h, x, row, col, direction, cross, edge_attr,
                       update_coords_mask, coords_range):
    """egnn_new.py:96-132: phi (and phi_x) per edge, trans = dir*tanh(phi)*range (+ cross*tanh(phi_x)*range),
    receiver-side segment sum, masked add."""
    z = torch.cat([h[row], h[col], edge_attr], dim=1)
    phi = _scalar_mlp3(sd, prefix + '.coord_mlp', z)
    trans = direction * torch.tanh(phi) * coords_range if cfg.tanh else direction * phi
    if not cfg.reflection_equivariant:
        phi_x = _scalar_mlp3(sd, prefix + '.cross_product_mlp', z)
        if cfg.tanh:
            phi_x = torch.tanh(phi_x) * coords_range
        trans = trans + cross * phi_x
    agg = segment_sum(trans, row, x.shape[0], cfg.normalization_factor, cfg.aggregation_method)
    if update_coords_mask is not None:
        agg = update_coords_mask * agg
    return x + agg


def sin_embedding(d2):
    """egnn_new.py:282-293 (``SinusoidsEmbeddingNew``, max_res=15, min_res=15/2000, div_factor=4): 6 frequencies
    2*pi*4^k/15, features [sin(f_k d) | cos(f_k d)] of d = sqrt(d^2 + 1e-8)."""
    n = int(math.log(15. / (15. / 2000.), 4)) + 1
    freq = 2 * math.pi * 4 ** torch.arange(n) / 15.
    emb = torch.sqrt(d2 + 1e-8) * freq[None, :].to(d2.device)
    return torch.cat((emb.sin(), emb.cos()), dim=-1)


def egnn_stack(sd, cfg, h, x, edges, update_coords_mask, batch_mask, edge_type_emb):
    """egnn_new.py:225-244 with the block body :163-184. ``coords_range`` passed to the blocks is
    the undivided 15.0 (egnn_new.py:197 computes /n_layers but :218 passes the raw value)."""
    row, col = edges[0], edges[1]
    d2_in, _ = radial_and_direction(x, row, col, 1)          # egnn_new.py:228 (default norm_constant)
    if cfg.sin_embedding:
        d2_in = sin_embedding(d2_in)                         # egnn_new.py:229-230
    edge_feat = d2_in if edge_type_emb is None else torch.cat([d2_in, edge_type_emb], dim=1)
    h = _linear(sd, 'egnn.embedding', h)
    coords_range = 15.0
    for k in range(cfg.n_layers):
        b = f'egnn.e_block_{k}'
        d2, direction = radial_and_direction(x, row, col, cfg.norm_constant)
        cross = None if cfg.reflection_equivariant else \
            cross_direction(x, row, col, batch_mask, cfg.norm_constant)
        if cfg.sin_embedding:
            d2 = sin_embedding(d2)                           # egnn_new.py:173-174
        edge_attr = torch.cat([d2, edge_feat], dim=1)
        for s in range(cfg.inv_sublayers):
            h = gcl(sd, f'{b}.gcl_{s}', cfg, h, row, col, edge_attr)
        x = equivariant_update(sd, f'{b}.gcl_equiv', cfg, h, x, row, col, direction, cross, edge_attr,
                               update_coords_mask, coords_range)
    h = _linear(sd, 'egnn.embedding_out', h)
    return h, x


def denoiser_forward(cfg, state_dict: Dict[str, torch.Tensor], xh_atoms, xh_residues, t,
                     mask_atoms, mask_residues, dtype=torch.float32,
                     return_edges: bool = False, device='cpu', edges=None):
    """``EGNNDynamics.forward`` (dynamics.py:87-167), eval mode, ``mode='egnn_dynamics'``.

    Returns ``(out_atoms [N_L,3+A], out_residues [N_P,3+R])`` on ``device`` (default CPU: the checker) in ``dtype``;
    raises ``ValueError('NaN detected in EGNN output')`` like dynamics.py:155-159.  ``device='cuda'`` runs the very same
    ATen op sequence on the GPU: that is bench.py's ``--impl reference-gpu`` arm ("the reference's own PyTorch graph on
    the GPU", SURVEY.md §8(d)), never a checker and never the product path.

    ``edges``: an int64 ``[2, E]`` edge list to evaluate on instead of ``build_edges`` (every edge must join two nodes of
    one graph).  A float64 evaluation decides the cut-offs on float64 distances, which can differ from an fp32 decision
    for pairs within a few ulp of a cut-off; passing the fp32 kernel's own edge list compares the two on the same graph."""
    if cfg.mode != 'egnn_dynamics':
        raise NotImplementedError('oracle covers mode=egnn_dynamics')
    sd = {k: v.detach().to(device, dtype) for k, v in state_dict.items()}
    xh_atoms = xh_atoms.detach().to(device, dtype)
    xh_residues = xh_residues.detach().to(device, dtype)
    t = t.detach().to(device, dtype)
    mask_atoms = mask_atoms.detach().to(device, torch.int64)
    mask_residues = mask_residues.detach().to(device, torch.int64)
    nd = cfg.n_dims
    n_lig = len(mask_atoms)

    with torch.no_grad():
        x_lig, h_lig = xh_atoms[:, :nd], xh_atoms[:, nd:]
        x_poc, h_poc = xh_residues[:, :nd], xh_residues[:, nd:]
        h = torch.cat((_mlp2(sd, 'atom_encoder', h_lig), _mlp2(sd, 'residue_encoder', h_poc)), dim=0)
        x = torch.cat((x_lig, x_poc), dim=0)
        mask = torch.cat([mask_atoms, mask_residues])
        if cfg.condition_time:
            if t.numel() == 1:                       # dynamics.py:105-107
                h_time = torch.full_like(h[:, 0:1], float(t.reshape(-1)[0]))
            else:                                    # dynamics.py:110
                h_time = t[mask]
            h = torch.cat([h, h_time], dim=1)
        if edges is None:
            edges = build_edges(cfg, mask_atoms, mask_residues, x_lig, x_poc)
        else:
            edges = edges.detach().to(device, torch.int64)
        assert torch.all(mask[edges[0]] == mask[edges[1]])       # dynamics.py:115
        emb = None
        if cfg.edge_embedding_dim:                                # dynamics.py:118-125
            etype = torch.zeros(edges.shape[1], dtype=torch.int64, device=edges.device)
            etype[(edges[0] < n_lig) & (edges[1] < n_lig)] = 1
            etype[(edges[0] >= n_lig) & (edges[1] >= n_lig)] = 2
            emb = sd['edge_embedding.weight'][etype]
        ucm = None if cfg.update_pocket_coords else torch.cat(
            (torch.ones_like(mask_atoms), torch.zeros_like(mask_residues))).unsqueeze(1).to(dtype)
        h_fin, x_fin = egnn_stack(sd, cfg, h, x, edges, ucm, mask, emb)
        vel = x_fin - x
        if cfg.condition_time:
            h_fin = h_fin[:, :-1]
        out_h_lig = _mlp2(sd, 'atom_decoder', h_fin[:n_lig])
        out_h_poc = _mlp2(sd, 'residue_decoder', h_fin[n_lig:])
        if torch.any(torch.isnan(vel)):
            raise ValueError('NaN detected in EGNN output')
        if cfg.update_pocket_coords:                              # dynamics.py:161-164 (joint mode)
            n_graphs = int(mask.max()) + 1
            vel = vel - segment_sum(vel, mask, n_graphs, None, 'mean')[mask]
        out = (torch.cat([vel[:n_lig], out_h_lig], dim=-1), torch.cat([vel[n_lig:], out_h_poc], dim=-1))
    if return_edges:
        return out + (edges,)
    return out
