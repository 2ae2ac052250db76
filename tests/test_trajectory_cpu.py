"""CPU: the planted cut-off boundary pairs have the float64 distances they claim, the float64 edge decision of the
trajectory tests reproduces the oracle's edge list where no pair is near a cut-off, and the oracle evaluated on a given
edge list equals the default call bit for bit."""
import math

import numpy as np
import pytest
import torch

from helpers import golden_cases, load_golden
from trajectory_cases import BLOCKS, OFFSETS, PLANT_CFG, candidate_pairs, compare_edges, planted_batch, ulp32
from oracle import egnn_oracle


def _pair_coords(inp, m):
    x = torch.cat((inp[0][:, :3], inp[1][:, :3]))
    return x[m['i']], x[m['j']]


def test_planted_pairs_have_claimed_distances():
    inp, meta = planted_batch()
    assert len(meta) == len(BLOCKS) * (2 + len(OFFSETS) * 5)
    rounded = generic = 0
    for m in meta:
        p, q = _pair_coords(inp, m)
        d = float((p.double() - q.double()).pow(2).sum().sqrt())
        cut, k = m['cut'], m['k']
        what = f"{m['block']} {m['kind']} k={k}"
        if k == 0:
            assert d == cut, what                              # exactly at the cut-off
        else:
            want = np.float32(cut)
            for _ in range(abs(k)):
                want = np.nextafter(want, np.float32(np.inf if k > 0 else -np.inf))
            assert m['claimed'] == float(want), what           # k float32 steps from the cut-off
            assert (d > cut) == (k > 0), what
        if m['kind'] in ('exact_axis', 'axis'):
            assert d == m['claimed'], what
            assert torch.count_nonzero(p - q) == 1, what        # along one axis
        else:
            assert abs(d - m['claimed']) <= ulp32(cut) / 8, f'{what}: {d!r} vs {m["claimed"]!r}'
            assert 10.0 <= float(p.double().norm()) <= 30.0, what
        if m['kind'] == 'generic':
            assert torch.count_nonzero(p - q) == 3, what        # generic direction
            generic += 1
            rounded += int(not torch.equal((p - q).double(), p.double() - q.double()))
    # in most generic pairs a float32 coordinate difference is not exact, so the kernel's d^2 carries rounding
    assert rounded >= generic // 2, (rounded, generic)


def test_planted_pairs_are_isolated():
    """One planted pair per graph: every other same-graph pair is a self-pair."""
    inp, meta = planted_batch()
    row, col, _ = candidate_pairs(inp[3], inp[4])
    off = row != col
    assert sorted(zip(row[off].tolist(), col[off].tolist())) == sorted(
        [(m['i'], m['j']) for m in meta] + [(m['j'], m['i']) for m in meta])


@pytest.mark.parametrize('case', golden_cases())
def test_float64_edge_decision_matches_oracle_edges(case):
    """The goldens keep every pair at least 2e-5 A from a cut-off, so the float64 decision of compare_edges must accept
    the oracle's (and the reference's) edge list with no pair in the band."""
    cfg, _, inp, _, edges = load_golden(case)
    n, in_band, _, bad = compare_edges(cfg, edges, inp[0][:, :3], inp[1][:, :3], inp[3], inp[4])
    assert not bad and in_band == 0 and n >= edges.shape[1]


def test_float64_edge_decision_on_planted_pairs():
    """compare_edges on the planted batch with the float64 decision itself as the edge list: nothing to report outside the
    band, and the band holds exactly the pairs within 4 ulp(cut)."""
    inp, meta = planted_batch()
    row, col, block = candidate_pairs(inp[3], inp[4])
    x = torch.cat((inp[0][:, :3], inp[1][:, :3])).double()
    d = (x[row] - x[col]).pow(2).sum(1).sqrt()
    cuts = torch.tensor([PLANT_CFG.edge_cutoff_ligand, PLANT_CFG.edge_cutoff_pocket, PLANT_CFG.edge_cutoff_interaction],
                        dtype=torch.float64)[block]
    keep = d <= cuts
    edges = torch.stack((row[keep], col[keep]))
    N = inp[0].shape[0] + inp[1].shape[0]
    edges = edges[:, torch.argsort(edges[0] * N + edges[1])]
    _, in_band, disagree, bad = compare_edges(PLANT_CFG, edges, inp[0][:, :3], inp[1][:, :3], inp[3], inp[4])
    assert not bad and disagree == 0
    dist = {(m['i'], m['j']): float((x[m['i']] - x[m['j']]).pow(2).sum().sqrt()) for m in meta}
    assert in_band == 2 * sum(1 for m in meta if abs(dist[m['i'], m['j']] - m['cut']) <= 4 * ulp32(m['cut']))
    assert in_band >= 2 * len(BLOCKS) * 2 * 6      # exact pairs and the +-1, +-2 ulp offsets at least


@pytest.mark.parametrize('case', golden_cases())
def test_oracle_on_given_edges_equals_default(case):
    cfg, sd, inp, _, _ = load_golden(case)
    edges = egnn_oracle.build_edges(cfg, inp[3], inp[4], inp[0][:, :3], inp[1][:, :3])
    want = egnn_oracle.denoiser_forward(cfg, sd, *inp)
    got = egnn_oracle.denoiser_forward(cfg, sd, *inp, edges=edges)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def test_oracle_on_given_edges_uses_them():
    """Dropping one edge changes the output: the given list is the one evaluated."""
    cfg, sd, inp, _, edges = load_golden('ragged_b3_l4')
    keep = torch.ones(edges.shape[1], dtype=torch.bool)
    keep[(edges[0] != edges[1]).nonzero()[0]] = False
    got = egnn_oracle.denoiser_forward(cfg, sd, *inp, edges=edges[:, keep])
    want = egnn_oracle.denoiser_forward(cfg, sd, *inp)
    assert not torch.equal(got[0], want[0])
    bad = edges.clone()
    bad[1, 0] = inp[0].shape[0] + inp[1].shape[0] - 1           # a pair of two different graphs
    with pytest.raises(AssertionError):
        egnn_oracle.denoiser_forward(cfg, sd, *inp, edges=bad)
