"""Shared definitions of the stress-shape denoiser cases (CPU structure / oracle tests and the GPU kernel tests).

The golden fixtures and the other parity tests use small, well-behaved graphs: no receiver there has more than 128 edges and
no receiver's edge segment spans three 128-row edge tiles.  The cases below go where real inputs go and the kernels'
bookkeeping is most delicate:

* receivers whose edges fill one or more whole 128-row tiles, both in CSR order (the fp32 FFMA edge kernels reduce per
  receiver in two 64-row halves of each tile) and in the virtual order padded to whole 4-row chunks (the wgmma edge kernels);
* ``aggregation_method='mean'`` with the receiver degree as the divisor at degree 256 next to degree 1;
* graphs without pocket nodes, without ligand atoms, a graph id with no nodes at all (its ``t`` entry still present) and a
  one-node graph, all in one batch.

``make_inputs`` is this module's own builder: ``synthetic.synthetic_denoiser_inputs`` divides by the pocket size, which is
undefined for a graph without pocket nodes.
"""
import torch

from diffsbdd_b200.config import DynamicsConfig
from diffsbdd_b200 import synthetic as syn

TILE = 128          # edge rows per tile of the edge kernels
CHUNK = 4           # receiver segments start at a multiple of this in the virtual edge order of the wgmma kernels

NO_CUTOFF = dict(edge_cutoff_ligand=None, edge_cutoff_pocket=None, edge_cutoff_interaction=None)

LADDER_SIZES = [1, 2, 3, 4, 5, 63, 64, 65, 127, 128, 129, 257]


def _ladder(n):
    """One graph of n nodes: about a third ligand atoms (at least one), the rest pocket nodes."""
    n_lig = max(1, round(n / 3))
    return n_lig, n - n_lig


# name -> dict(cfg, graphs = [(n_lig, n_pocket) per graph id], seed, wseed, expect = structure the case must have)
#   expect: min_max_deg (largest receiver degree at least), csr_cross / virt_cross (receivers whose segment crosses a
#   128-row boundary in CSR / virtual order: at least 1), span3 (receivers whose virtual segment touches >= 3 tiles: at
#   least 1), min_deg_lig (every ligand atom has at least this degree), deg1 (a receiver of degree exactly 1), empty
#   (graph ids with no node), no_pocket / no_ligand (graph ids with ligand atoms only / pocket nodes only), edge_types
#   (ligand-ligand, pocket-pocket and ligand-pocket edges all present), min_units (more than this many 128-row units of
#   the virtual edge order in the GCL and in the coordinate edge kernel)
CASES = {
    # conditional, no cut-offs: degree = graph size for every node
    'ladder_h128': dict(cfg=DynamicsConfig(hidden_nf=128, joint_nf=32, n_layers=2, **NO_CUTOFF),
                        graphs=[_ladder(n) for n in LADDER_SIZES], seed=41, wseed=41,
                        expect=dict(min_max_deg=257, csr_cross=True, virt_cross=True, span3=True, deg1=True, no_pocket=[0])),
    'ladder_h256': dict(cfg=DynamicsConfig(hidden_nf=256, n_layers=2, **NO_CUTOFF),
                        graphs=[_ladder(n) for n in LADDER_SIZES], seed=42, wseed=42,
                        expect=dict(min_max_deg=257, csr_cross=True, virt_cross=True, span3=True, deg1=True, no_pocket=[0])),
    # configs/crossdock_fullatom_cond.yml dims (no ligand cut-off, 5 A pocket / interaction cut-offs): a 150-atom ligand in a
    # 350-atom pocket at full-atom density, next to one graph of the configs[2] shape
    'dense_cond': dict(cfg=DynamicsConfig(n_layers=3), graphs=[(150, 350), (25, 175)], seed=47, wseed=43,
                       expect=dict(min_max_deg=151, csr_cross=True, virt_cross=True, span3=True, min_deg_lig=25)),
    # joint model, fully connected ~300-node graph: cross-product centroid and velocity-mean removal over a large graph
    'joint_fc_h192': dict(cfg=DynamicsConfig(hidden_nf=192, joint_nf=64, n_layers=2, update_pocket_coords=True,
                                             reflection_equivariant=False, **NO_CUTOFF),
                          graphs=[(100, 200), (6, 11)], seed=44, wseed=44,
                          expect=dict(min_max_deg=300, csr_cross=True, virt_cross=True, span3=True)),
    'joint_fc_reflect_h192': dict(cfg=DynamicsConfig(hidden_nf=192, joint_nf=64, n_layers=2, update_pocket_coords=True,
                                                     reflection_equivariant=True, **NO_CUTOFF),
                                  graphs=[(100, 200), (6, 11)], seed=45, wseed=45,
                                  expect=dict(min_max_deg=300, csr_cross=True, virt_cross=True, span3=True)),
    # 'mean' aggregation: the divisor is the receiver degree, 256 and 1 in one batch
    'mean_h256': dict(cfg=DynamicsConfig(n_layers=2, aggregation_method='mean', **NO_CUTOFF),
                      graphs=[(86, 170), (1, 0)], seed=46, wseed=46,
                      expect=dict(min_max_deg=256, csr_cross=True, virt_cross=True, span3=True, deg1=True, no_pocket=[1])),
    # degenerate structure: one ligand atom without pocket, an empty graph id, pocket without ligand, an ordinary graph and a
    # trailing empty graph id; H=64 runs the fp32 FFMA kernels only
    'degenerate_h64': dict(cfg=DynamicsConfig(hidden_nf=64, joint_nf=16, n_layers=2),
                           graphs=[(1, 0), (0, 0), (0, 23), (9, 31), (0, 0)], seed=47, wseed=47,
                           expect=dict(deg1=True, empty=[1, 4], no_pocket=[0], no_ligand=[2])),
    'degenerate_h128': dict(cfg=DynamicsConfig(hidden_nf=128, joint_nf=32, n_layers=2),
                            graphs=[(1, 0), (0, 0), (0, 23), (9, 31), (0, 0)], seed=48, wseed=48,
                            expect=dict(deg1=True, empty=[1, 4], no_pocket=[0], no_ligand=[2])),
    'degenerate_joint_mean_h128': dict(cfg=DynamicsConfig(hidden_nf=128, joint_nf=32, n_layers=2, update_pocket_coords=True,
                                                          aggregation_method='mean'),
                                       graphs=[(1, 0), (0, 0), (0, 23), (9, 31), (0, 0)], seed=49, wseed=49,
                                       expect=dict(deg1=True, empty=[1, 4], no_pocket=[0], no_ligand=[2])),
    # edge-type table at H=128 without the attention gate or tanh (the only tensor-core kernels that read the table at that
    # width, and the gate = 1 / untanh'd branches of the edge epilogues); default cut-offs give all three edge types, and
    # 60-atom ligands give both edge kernels more 128-row units than the H100's 132 SMs (~290 GCL, ~160 coordinate units)
    'tb_noatt_notanh_h128': dict(cfg=DynamicsConfig(hidden_nf=128, joint_nf=32, n_layers=2, edge_embedding_dim=8,
                                                    attention=False, tanh=False),
                                 graphs=[(60, 150)] * 4, seed=57, wseed=57,
                                 expect=dict(min_max_deg=80, csr_cross=True, virt_cross=True, edge_types=True,
                                             min_units=132)),
}

# ligand rows [0, n) + pocket rows of the 257-node ladder graph, run alone and inside its batch
LADDER_BIG = LADDER_SIZES.index(257)


def math_modes(cfg):
    """Every arithmetic path the width supports: the tensor-core kernels exist for hidden_nf 128, 192 and 256."""
    return ['fp32', '3xtf32', '3xfp16'] if cfg.hidden_nf in (128, 192, 256) else ['fp32']


def make_inputs(cfg, graphs, seed, density=0.045, norm_values=(1.0, 4.0), lig_sigma=1.0):
    """``EGNNDynamics.forward`` arguments (CPU) for graphs given as (n_lig, n_pocket) per graph id; either count may be 0.

    Pocket: ``synthetic.synthetic_pocket`` points (uniform in a ball at ``density``), normalised.  Ligand: ~ N(pocket COM,
    lig_sigma), then the ligand COM is removed from the ligand and the pocket of its graph, as the conditional sampler does
    (conditional_model.py:151-158).  A graph without pocket nodes has its ligand around the origin; a graph without ligand
    atoms keeps its pocket as placed.  ``t`` is [n_graphs, 1] and has an entry for every graph id, empty ones included."""
    n_lig = [a for a, _ in graphs]
    n_poc = [b for _, b in graphs]
    B = len(graphs)
    pocket = syn.synthetic_pocket(cfg, n_poc, seed, density)
    g = torch.Generator().manual_seed(1000 + seed)
    mask_res = pocket['mask']
    mask_at = torch.repeat_interleave(torch.arange(B), torch.tensor(n_lig, dtype=torch.int64))
    x_p = pocket['x'].double() / norm_values[0]
    h_p = pocket['one_hot'].double() / norm_values[1]
    cnt_p = torch.tensor(n_poc, dtype=torch.float64).clamp(min=1)[:, None]
    com = torch.zeros((B, 3), dtype=torch.float64).index_add_(0, mask_res, x_p) / cnt_p
    z = torch.randn((len(mask_at), 3 + cfg.atom_nf), generator=g, dtype=torch.float64) * lig_sigma
    z[:, :3] += com[mask_at]
    cnt_l = torch.tensor(n_lig, dtype=torch.float64).clamp(min=1)[:, None]
    lig_mean = torch.zeros((B, 3), dtype=torch.float64).index_add_(0, mask_at, z[:, :3]) / cnt_l
    z[:, :3] -= lig_mean[mask_at]
    x_p = x_p - lig_mean[mask_res]
    t = torch.rand((B, 1), generator=g, dtype=torch.float64)
    return (z.to(torch.float32), torch.cat([x_p, h_p], 1).to(torch.float32), t.to(torch.float32),
            mask_at, mask_res.to(torch.int64))


def case_inputs(name):
    """(cfg, state_dict, inputs) of a case."""
    c = CASES[name]
    return c['cfg'], syn.synthetic_state_dict(c['cfg'], c['wseed']), make_inputs(c['cfg'], c['graphs'], c['seed'])


def single_graph_inputs(inp, g):
    """The forward arguments of graph g of a batch on its own (graph id 0)."""
    sa, sr = inp[3] == g, inp[4] == g
    return (inp[0][sa], inp[1][sr], inp[2][g:g + 1], torch.zeros(int(sa.sum()), dtype=torch.int64),
            torch.zeros(int(sr.sum()), dtype=torch.int64))


def edge_stats(edges, n_nodes, tile=TILE, chunk=CHUNK):
    """What the edge kernels' per-receiver reduction depends on, from a row-sorted [2, E] edge list.

    deg: per-receiver degree.  A receiver's segment is [start, start + len) in the CSR edge order (len = deg) or in the
    virtual order, where every segment is padded to a multiple of ``chunk`` rows (len = ceil(deg / chunk) * chunk).
    csr_cross / virt_cross: receivers whose segment crosses a multiple of ``tile``; csr_span3 / virt_span3: receivers whose
    segment touches three tiles or more."""
    row = edges[0]
    assert row.numel() == 0 or bool((row[1:] >= row[:-1]).all()), 'edge list must be sorted by receiver'
    deg = torch.bincount(row, minlength=n_nodes)
    out = {'deg': deg, 'max_deg': int(deg.max()) if n_nodes else 0}
    for name, seg in (('csr', deg), ('virt', (deg + chunk - 1) // chunk * chunk)):
        end = torch.cumsum(seg, 0)
        start = end - seg
        live = seg > 0
        tiles = torch.where(live, (end - 1) // tile - start // tile + 1, torch.zeros_like(seg))
        out[name + '_cross'] = int((tiles >= 2).sum())
        out[name + '_span3'] = int((tiles >= 3).sum())
    return out


def max_abs(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).abs().max()) if a.numel() else 0.0


def column_errors(got, want):
    """Max-abs error of (vel, h) columns over the ligand and pocket outputs; got/want = (out_atoms, out_residues)."""
    vel = max(max_abs(got[0][:, :3], want[0][:, :3]), max_abs(got[1][:, :3], want[1][:, :3]))
    h = max(max_abs(got[0][:, 3:], want[0][:, 3:]), max_abs(got[1][:, 3:], want[1][:, 3:]))
    return vel, h

