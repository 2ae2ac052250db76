"""CPU: the per-launch test hooks and the float64 launch restatements (tests/launch_cases.py).

* dsb_workspace_region: the regions of the forward's workspace are disjoint, 256-byte aligned and have the sizes the
  header states, for several configurations in both modes (that they lie inside dsb_dynamics_workspace_bytes needs a
  module, i.e. a GPU: tests/test_gpu_launches.py);
* the restatements chained launch by launch (launch_cases.emulate) reproduce the float64 oracle of the whole forward, so
  they restate the reference algebra and not something else;
* an fp32 evaluation of every launch stays inside the launch's worst-case bound (the bound is not too tight);
* the binade-sweep case has the operand ranges it is built for.
"""
import ctypes as C

import pytest
import torch

import launch_cases as lc
from helpers import load_golden, assert_close
from stress_cases import case_inputs
from diffsbdd_b200 import _build, _native
from diffsbdd_b200.config import DynamicsConfig, FULLATOM_COND, FULLATOM_JOINT
from diffsbdd_b200.dynamics import EGNNDynamics
from oracle import egnn_oracle


@pytest.fixture(scope='module')
def lib():
    _build.build()
    return _native.load(build_if_missing=False)


REGION_CFGS = [FULLATOM_COND, FULLATOM_JOINT, DynamicsConfig(hidden_nf=64, joint_nf=16, n_layers=2),
               DynamicsConfig(hidden_nf=192, reflection_equivariant=True, edge_embedding_dim=8)]
SIZES = [(25 * 64, 175 * 64, 64, 64 * 200 ** 2), (1, 0, 1, 1), (30, 41, 5, 900), (0, 7, 3, 49)]


@pytest.mark.parametrize('det', [0, 1])
@pytest.mark.parametrize('ci', range(len(REGION_CFGS)))
def test_workspace_regions_disjoint_inside_and_sized(lib, ci, det):
    cfg = REGION_CFGS[ci]
    net = EGNNDynamics.from_config(cfg)
    ccfg = net._c_config()
    H, nm = cfg.hidden_nf, 1 if cfg.reflection_equivariant else 2
    for NL, NP, B, ecap in SIZES:
        N = NL + NP
        reg = _native.workspace_regions(ccfg, det, NL, NP, B, ecap)
        assert set(reg) == set(_native.WS_REGIONS)
        spans = sorted((o, o + b, k) for k, (o, b) in reg.items() if b > 0)
        for (a0, a1, ka), (b0, b1, kb) in zip(spans, spans[1:]):
            assert a1 <= b0, f'{ka} [{a0}, {a1}) overlaps {kb} [{b0}, {b1})'
        for k, (o, b) in reg.items():
            assert o % 256 == 0, k
        for k in ('x_in', 'x_ping', 'x_pong', 'xagg'):
            assert reg[k][1] == 16 * (N + 1), k
        for k in ('h', 'agg'):
            assert reg[k][1] == 4 * (N + 1) * H, k
        assert reg['hT'][1] == 4 * (N + 257) * H
        assert reg['P'][1] == 4 * (N + 1) * 6 * H and (2 * nm + 2) * H <= 6 * H
        assert reg['erow'][1] == reg['ecol'][1] == reg['ed0'][1] == 4 * (ecap + 1)
        assert reg['vmap'][1] == 4 * (ecap + 3 * N + 1)
        assert reg['cent'][1] == reg['velmean'][1] == 16 * (B + 1)
        assert (reg['part'][1] > 0) == bool(det)


def test_workspace_region_rejects_bad_arguments(lib):
    ccfg = EGNNDynamics.from_config(FULLATOM_COND)._c_config()
    off, nb = C.c_int64(), C.c_int64()
    assert lib.dsb_workspace_region(C.byref(ccfg), 0, 10, 10, 1, 400, len(_native.WS_REGIONS), C.byref(off), C.byref(nb)) == -1
    assert lib.dsb_workspace_region(C.byref(ccfg), 0, -1, 10, 1, 400, 0, C.byref(off), C.byref(nb)) == -1
    ccfg.hidden_nf = 100
    assert lib.dsb_workspace_region(C.byref(ccfg), 0, 10, 10, 1, 400, 0, C.byref(off), C.byref(nb)) == -2
    assert lib.dsb_dynamics_set_stop_after(None, 3) == -1


def test_op_sequence_counts():
    """The restated operation order has the forward's launch count (DESIGN.md: 44 at configs[2], 56 deterministic)."""
    for det, want in ((False, 44), (True, 56)):
        ops = lc.op_sequence(FULLATOM_COND, det)
        assert sum(not o.kind.startswith('memset') for o in ops) == want
    units = lc.launch_units(FULLATOM_JOINT, True)
    assert [u[2].kind for u in units][:3] == ['prep', 'centroid', 'g1']
    assert units[-1][2].kind == 'velmean' and units[-1][1] == len(lc.op_sequence(FULLATOM_JOINT, True))


EMU_CASES = ['emb8_h256_l3', 'joint_emb8_sub2_reflect_h256_l2', 'mean_h256_l3', 'joint_b2_h128_l5', 'moad_emb8_h192_l3']


@pytest.mark.parametrize('name', EMU_CASES + ['degenerate_joint_mean_h128', 'joint_fc_h192', 'tb_noatt_notanh_h128', 'sweep'])
def test_restatements_chain_to_the_oracle(name):
    if name == 'sweep':
        cfg, sd, inp = lc.binade_sweep_case()
    elif name in EMU_CASES:
        cfg, sd, inp = load_golden(name)[:3]
    else:
        cfg, sd, inp = case_inputs(name)
    o64 = egnn_oracle.denoiser_forward(cfg, sd, *inp, dtype=torch.float64)
    e64 = lc.emulate(cfg, sd, inp, dtype=torch.float64)
    for a, b in zip(e64, o64):
        assert_close(a, b, f'{name}: fp64 restatements vs fp64 oracle', atol=1e-9, rtol=1e-9)
    if name != 'sweep':
        e32 = lc.emulate(cfg, sd, inp, dtype=torch.float32)
        for a, b in zip(e32, o64):
            assert_close(a, b, f'{name}: fp32 restatements vs fp64 oracle')


@pytest.mark.parametrize('name', ['emb8_h256_l3', 'joint_emb8_sub2_reflect_h256_l2', 'moad_emb8_h192_l3', 'sweep'])
def test_fp32_launches_inside_their_bounds(name):
    """Teacher-forced on the fp32 chain: every launch's fp32 evaluation is within its float64 worst-case bound."""
    if name == 'sweep':
        cfg, sd, inp = lc.binade_sweep_case()
    else:
        cfg, sd, inp = load_golden(name)[:3]
    S = lc.initial_state(cfg, inp, torch.float32)
    r32 = lc.Restater(cfg, sd, inp, 0, torch.float32)
    r64 = lc.Restater(cfg, sd, inp, 0, torch.float64)
    worst = 0.0
    for _, _, op in lc.launch_units(cfg, False):
        o32, o64 = r32.run(op, S), r64.run(op, S)
        for k, (v64, b64, *_) in o64.items():
            if b64 is None:
                continue
            err = (o32[k][0].double() - v64).abs()
            ratio = float((err / (b64 + 1e-300)).max())
            worst = max(worst, ratio)
            assert ratio <= 1.0, f'{name} {op.kind} l{op.layer} {k}: fp32 error {ratio:.2f} x bound'
        lc.apply(S, o32)
    print(f'{name}: largest fp32 error / bound {worst:.3f}')


def test_binade_sweep_operand_ranges():
    cfg, sd, inp = lc.binade_sweep_case()
    r = lc.sweep_operand_ranges(cfg, sd, inp)
    for k, (lo, hi) in r.items():
        print(k, f'{lo:.2e} {hi:.2e}')
        assert lo <= 2.0 ** -18, (k, lo)             # reaches well into the fp16 subnormal range (< 2^-14)
        assert 2.0 ** 12 <= hi < 60000.0, (k, hi)    # large, and below the fp16 limit 65504
