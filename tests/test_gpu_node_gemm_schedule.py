"""GPU: the tensor-core node GEMMs (g1 - g4) at the row counts where their tile loop has edge cases, checked launch by launch
against the float64 restatements and bounds of tests/launch_cases.py, in deterministic mode.

Row counts M = N (nodes) and ligand counts NL of the cases (128-row output tiles, 64 rows per MMA warpgroup):

    case        M     M mod 64   64-row blocks   tiles   NL    (g4 dead region starts at ceil(NL / 128) * 128)
    m50         50    50         1               1       13    128: no dead tile
    m193        193   1          4               2       70    128
    m319        319   63         5               3       150   256
    m384        384   0          6               3       100   128

Every case has fewer tiles than the H100 has SMs, the last tile is partial in all but m384, and no NL is a multiple of 64.
The merged first-layer GEMM g4 skips the receiver-side coordinate columns of pocket rows at 128-row tile granularity
(``dead_p_mask``): with P pre-filled with a sentinel, every element outside the mask must be written and every element
inside it left untouched.  Widths 128, 192 and 256, math modes 15 (3xFP16) and 7 (3xTF32).
"""
import pytest
import torch

import launch_cases as lc
import test_gpu_launches as tl
from diffsbdd_b200 import synthetic as syn
from diffsbdd_b200.config import FULLATOM_COND

pytestmark = pytest.mark.gpu

SHAPES = {                     # (ligand atoms per graph, pocket nodes per graph)
    'm50': ([6, 7], [20, 17]),
    'm193': ([30, 40], [60, 63]),
    'm319': ([70, 80], [90, 79]),
    'm384': ([45, 55], [140, 144]),
}
WIDTHS = (128, 192, 256)
MODES = (15, 7)
GEMMS = ('g1', 'g2', 'g3', 'g4')
SENTINEL = 0x7FC0DEAD          # a NaN no kernel writes


def make_case(shape, H):
    cfg = FULLATOM_COND.with_(hidden_nf=H, n_layers=2)
    lig, poc = SHAPES[shape]
    return cfg, syn.synthetic_state_dict(cfg, 11), syn.synthetic_denoiser_inputs(cfg, lig, poc, seed=5)


def runner(monkeypatch, shape, H, mode):
    name = f'{shape}_h{H}'
    case = make_case(shape, H)
    monkeypatch.setitem(tl.CASES, name, lambda: case)
    return tl.Runner(name, mode, True)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('H', WIDTHS)
@pytest.mark.parametrize('shape', sorted(SHAPES))
def test_node_gemms_against_float64(monkeypatch, shape, H, mode):
    r = runner(monkeypatch, shape, H, mode)
    n_checked = 0
    for i, j, op in lc.launch_units(r.cfg, True):
        if op.kind not in GEMMS:
            continue
        r.check_unit(op, r.state(r.snapshot(i)), r.state(r.snapshot(j)))
        n_checked += 1
    assert n_checked == 1 + 3 * r.cfg.n_layers
    assert not r.failures, '\n'.join(r.failures)


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('H', WIDTHS)
@pytest.mark.parametrize('shape', sorted(SHAPES))
def test_g4_writes_exactly_the_live_tiles(monkeypatch, shape, H, mode):
    r = runner(monkeypatch, shape, H, mode)
    ops = lc.op_sequence(r.cfg, True)
    k = next(i for i, op in enumerate(ops) if op.kind == 'g4')
    off, nbytes = r.regions['P']
    r.net._workspace[off:off + nbytes].view(torch.int32).fill_(SENTINEL)
    tl.run_stopped(r.net, r.inp, k + 1)
    P = r.state(r.net._workspace)['P']
    bits = P.contiguous().view(torch.int32).cpu()
    dead = lc.dead_p_mask(r.cfg, r.dm, mode, P.shape[1])      # g4 of block 0 writes every column of P
    live_rows_end = -(-r.dm.NL // 128) * 128
    assert dead.any() == (live_rows_end < r.dm.N)
    assert bool((bits[dead] == SENTINEL).all()), 'a skipped tile of P was written'
    assert bool((bits[~dead] != SENTINEL).all()), 'an element of a live tile of P was not written'
    assert torch.isfinite(P[~dead.cuda()]).all()
