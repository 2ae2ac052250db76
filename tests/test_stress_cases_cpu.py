"""CPU: the stress-shape cases (tests/stress_cases.py) have the structure they are meant to exercise, and the fp32 oracle meets
the project tolerance against the fp64 oracle on every one of them, so an fp32 implementation can too."""
import pytest
import torch

from helpers import assert_close, ATOL, RTOL
from stress_cases import CASES, CHUNK, TILE, case_inputs, edge_stats, column_errors
from diffsbdd_b200 import synthetic as syn
from oracle import egnn_oracle


@pytest.mark.parametrize('name', sorted(CASES))
def test_case_structure(name):
    spec, ex = CASES[name], CASES[name]['expect']
    cfg, sd, inp = case_inputs(name)
    xa, xr, t, ma, mr = inp
    B = len(spec['graphs'])
    assert t.shape == (B, 1)
    assert torch.equal(torch.bincount(ma, minlength=B), torch.tensor([a for a, _ in spec['graphs']]))
    assert torch.equal(torch.bincount(mr, minlength=B), torch.tensor([b for _, b in spec['graphs']]))
    assert syn.min_cutoff_margin(cfg, xa, xr, ma, mr) > 1e-4
    edges = egnn_oracle.build_edges(cfg, ma, mr, xa[:, :3], xr[:, :3])
    st = edge_stats(edges, len(ma) + len(mr))
    deg = st['deg']
    assert int(deg.min()) >= 1                                   # every node has its self edge
    assert st['max_deg'] >= ex.get('min_max_deg', 0)
    if ex.get('csr_cross'):
        assert st['csr_cross'] > 0
    if ex.get('virt_cross'):
        assert st['virt_cross'] > 0
    if ex.get('span3'):
        assert st['csr_span3'] > 0 and st['virt_span3'] > 0
    if 'min_deg_lig' in ex:
        assert int(deg[:len(ma)].min()) >= ex['min_deg_lig']
    if ex.get('deg1'):
        assert int((deg == 1).sum()) > 0
    if cfg.edge_cutoff_ligand is None and cfg.edge_cutoff_pocket is None and cfg.edge_cutoff_interaction is None:
        size = torch.bincount(torch.cat([ma, mr]), minlength=B)
        assert torch.equal(deg, size[torch.cat([ma, mr])])       # fully connected graphs: degree = graph size
    if ex.get('edge_types'):
        NL, er, ec = len(ma), edges[0], edges[1]
        assert bool(((er < NL) & (ec < NL)).any()) and bool(((er >= NL) & (ec >= NL)).any())
        assert bool(((er < NL) != (ec < NL)).any())
    if 'min_units' in ex:
        vdeg = (deg + CHUNK - 1) // CHUNK * CHUNK
        n_coord = len(deg) if cfg.update_pocket_coords else len(ma)
        for what, rows in (('GCL', vdeg), ('coordinate', vdeg[:n_coord])):
            units = -(-int(rows.sum()) // TILE)
            assert units > ex['min_units'], f'{what} edge kernel: {units} units'
    for g in ex.get('empty', []):
        assert not bool((ma == g).any()) and not bool((mr == g).any())
    for g in ex.get('no_pocket', []):
        assert bool((ma == g).any()) and not bool((mr == g).any())
    for g in ex.get('no_ligand', []):
        assert not bool((ma == g).any()) and bool((mr == g).any())


def test_ladder_counts():
    """The ladder batch as designed: N = 848 nodes, E = sum of squared graph sizes, the 257-node graph's receivers all span
    three tiles."""
    cfg, sd, inp = case_inputs('ladder_h256')
    edges = egnn_oracle.build_edges(cfg, inp[3], inp[4], inp[0][:, :3], inp[1][:, :3])
    st = edge_stats(edges, len(inp[3]) + len(inp[4]))
    assert len(inp[3]) + len(inp[4]) == 848 and edges.shape[1] == 127548
    assert st['virt_span3'] >= 257 and st['virt_cross'] > 700


def test_edge_stats_counts_by_hand():
    # receivers of degree 130, 1, 126, 300 in CSR order: segments [0,130) [130,131) [131,257) [257,557)
    row = torch.repeat_interleave(torch.arange(4), torch.tensor([130, 1, 126, 300]))
    st = edge_stats(torch.stack([row, torch.zeros_like(row)]), 4)
    assert st['deg'].tolist() == [130, 1, 126, 300] and st['max_deg'] == 300
    assert st['csr_cross'] == 3 and st['csr_span3'] == 1         # tiles 0-1, 1-2 and 2-4
    # virtual order pads to 132, 4, 128, 300: [0,132) [132,136) [136,264) [264,564)
    assert st['virt_cross'] == 3 and st['virt_span3'] == 1       # tiles 0-1, 1-2 and 2-4


@pytest.mark.parametrize('name', sorted(CASES))
def test_fp32_oracle_meets_tolerance_against_fp64(name):
    """The floor the GPU error budget is measured against (tests/test_gpu_stress_shapes.py), and proof that the project
    tolerance can be met in fp32 at these degrees."""
    cfg, sd, inp = case_inputs(name)
    o32 = egnn_oracle.denoiser_forward(cfg, sd, *inp)
    o64 = egnn_oracle.denoiser_forward(cfg, sd, *inp, dtype=torch.float64)
    assert all(torch.isfinite(o).all() for o in o64)
    assert_close(o32[0], o64[0], f'{name} ligand fp32 vs fp64', atol=ATOL, rtol=RTOL)
    assert_close(o32[1], o64[1], f'{name} pocket fp32 vs fp64', atol=ATOL, rtol=RTOL)
    vel, h = column_errors(o32, o64)
    print(f'{name}: fp32 oracle vs fp64 max abs err vel {vel:.2e} h {h:.2e}')
    if not cfg.update_pocket_coords:
        assert torch.count_nonzero(o64[1][:, :3]) == 0
