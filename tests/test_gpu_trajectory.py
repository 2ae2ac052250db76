"""GPU: the production sampler checked step by step along recorded 500-step trajectories, and the edge cut-off at its
boundary.

The trajectories (tests/trajectory_cases.py) are the production configurations run by the production graph engine in
deterministic mode: ``ConditionalDDPM.sample_given_pocket`` with the FULLATOM_COND denoiser (H=256, 6 layers, 3xFP16) on
the configs[2] pocket batch (64 x (25 + 175) atoms), and the joint ``EnVariationalDiffusion.sample`` with FULLATOM_JOINT
(H=128, 5 layers) on 16 graphs of 25 + 175 nodes; T = 500, polynomial_2 schedule.  Every check feeds the kernels and the
references the same recorded fp32 state ("teacher forcing"), so each comparison is one step or one call, well posed, with
no amplification along the chain.  A free-running chain is not compared with anything: two correct fp32 implementations
can cross an edge cut-off on different steps, and their chains then differ by whole messages.

* The recorded run gives the same bits as an unmodified sampler call with the same seed.
* Step tables, every step: t = (s+1)/T, and the coefficients the graph read equal the eager step's, bit for bit.
* Fused update, every step: the native denoiser called eagerly on the recorded input plus the fused update kernel on the
  recorded noise reproduce the replay's output bit for bit; that output meets ddpm_cases.assert_fp64_bound against the
  float64 evaluation of the eager update ops.
* Denoiser against float64, 36 calls (the first 8 reverse steps, every 25th, the last 8, and the t = 0 call of
  sample_p_xh_given_z0), in 3xFP16, 3xTF32 and fp32 (deterministic) and 3xFP16 (default mode): helpers.ATOL/RTOL against
  the float64 oracle, and vel and h errors each at most K = 10 x the fp32 oracle's own error + 1e-7 (the criteria of
  test_gpu_stress_shapes.py).  Both oracles run on the GPU on the native edge list (TF32 off for the fp32 one): near a
  cut-off a float64 distance can decide a pair differently from the fp32 kernel, and that is a property of the cut-off,
  not a kernel error.
* Edge list, every step: get_edges agrees with the decision d <= cut on float64 distances of the same fp32 coordinates for
  every same-graph pair more than 4 ulp(cut) from its cut-off.
* Planted boundary pairs (cut-offs 3 / 4 / 7 A): pairs exactly at a cut-off are kept; axis-aligned pairs, whose fp32
  distance is exact, are decided exactly; generic pairs more than 4 ulp(cut) inside are kept and more than 4 ulp(cut)
  outside are dropped; the forward pass uses the edges get_edges returns.

Why 4 ulp.  The kernel keeps a pair iff fp32 sqrtf(dx*dx + dy*dy + dz*dz) <= cut.  Each coordinate difference rounds with
relative error at most u = 2^-24, each square adds one rounding, the sum two (fewer with FMA contraction) and the
correctly rounded sqrtf one more, so to first order |sqrtf(d2) - d| <= (3u + 2u) / 2 * d + u * d = 3.5 u d < 3.5 ulp(d).
Pairs more than 4 ulp(cut) from the cut-off are therefore decided as float64 decides them.

The project tolerance against fp64 is asserted on the column groups (ligand / pocket x vel / h) where the fp32 oracle's
own error is within a tenth of it, the headroom the tolerance was set with.  Real sampler states leave less: past the
first steps the fp32 oracle's vel error reaches 1-4e-5 on the conditional ligand and up to 2.6e-4 on the joint model
(the synthetic joint weights spread each graph out: 636k edges at t = 1, 12.8k from mid-chain on), and its h error
2-7e-6 on the conditional model, where 3xTF32 (h ratio up to 6) reaches 2.5e-5.  There the K ratio is the criterion.

Measured on one H100 80GB HBM3 at a 700 W power limit, ratios err_native / err_fp32_oracle, vel / h, maximum over the
calls of each group (early: the first 8 steps; middle: every 25th; late: the last 8 and the t = 0 call).  The ratios
move by a few tenths between runs (the default mode's atomics; the oracles' cuBLAS kernels):

    model  group    3xfp16        3xtf32        fp32          3xfp16 default
    cond   early    1.91 / 3.00   3.84 / 4.45   1.10 / 1.84   2.87 / 2.56
    cond   middle   1.48 / 3.14   2.66 / 5.92   1.27 / 0.75   1.43 / 3.24
    cond   late     2.01 / 2.77   2.37 / 5.48   1.66 / 1.05   1.83 / 2.96
    joint  early    2.62 / 2.59   5.05 / 3.21   1.22 / 2.45   2.62 / 3.04
    joint  middle   1.18 / 1.72   1.93 / 3.35   1.01 / 1.27   1.15 / 1.67
    joint  late     1.37 / 1.61   1.37 / 2.75   1.37 / 0.76   1.37 / 1.61

Edge lists along the trajectories: 384 pair-states of the conditional run lie within 4 ulp of a cut-off (40 of them
decided differently from float64); none in the joint run.  Of the 156 planted pairs, 60 generic ones lie within the band.
The file takes about 40 s on that GPU.
"""
import time
from types import SimpleNamespace

import pytest
import torch

from ddpm_cases import assert_fp64_bound
from repaint_cases import joint_step_coefficients
from helpers import ATOL, RTOL, assert_close
from stress_cases import column_errors
from trajectory_cases import (COND_SEED, JOINT_LIG, JOINT_POC, JOINT_SEED, PLANT_CFG, T, candidate_pairs, compare_edges,
                              full_pocket, joint_update, joint_update_ref, ligand_update, ligand_update_ref, make_ddpm,
                              planted_batch, record_conditional, record_joint, ulp32)
from diffsbdd_b200 import synthetic as syn
from diffsbdd_b200.config import FULLATOM_COND, FULLATOM_JOINT
from diffsbdd_b200.dynamics import EGNNDynamics
from oracle import egnn_oracle

pytestmark = pytest.mark.gpu

K = 10.0
FLOOR = 1e-7
DELTA_ULPS = 4
# reverse steps k (s = T-1-k) checked against float64: the first 8, every 25th, the last 8; k = T is the t = 0 call
SELECTED = list(range(8)) + list(range(25, T - 8, 25)) + list(range(T - 8, T)) + [T]
# (label, math mode, deterministic)
MODES = [('3xfp16', '3xfp16', True), ('3xtf32', '3xtf32', True), ('fp32', 'fp32', True), ('3xfp16 dflt', '3xfp16', False)]


@pytest.fixture(scope='module', autouse=True)
def no_tf32():
    """The fp32 oracle on the GPU is the fp32 baseline only with TF32 off."""
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


@pytest.fixture(scope='module', params=['cond', 'joint'])
def traj(request):
    joint = request.param == 'joint'
    cfg = FULLATOM_JOINT if joint else FULLATOM_COND
    ddpm = make_ddpm(cfg, joint)
    t0 = time.time()
    if joint:
        n_lig, n_poc = torch.tensor(JOINT_LIG).cuda(), torch.tensor(JOINT_POC).cuda()
        rec = record_joint(ddpm, n_lig, n_poc)
        torch.manual_seed(JOINT_SEED)
        plain = ddpm.sample(len(JOINT_LIG), n_lig, n_poc, device='cuda')
    else:
        pocket, n_lig = full_pocket()
        rec = record_conditional(ddpm, pocket, n_lig)
        torch.manual_seed(COND_SEED)
        plain = ddpm.sample_given_pocket({k: v.clone() for k, v in pocket.items()}, n_lig)
    torch.cuda.synchronize()
    print(f'\n[{request.param}] recorded + unmodified 500-step runs: {time.time() - t0:.1f} s')
    yield SimpleNamespace(name=request.param, joint=joint, cfg=cfg, sd=syn.synthetic_state_dict(cfg, 0), ddpm=ddpm,
                          rec=rec, plain=plain, lm=rec['lig_mask'], pm=rec['pocket_mask'], n=rec['t'][0].shape[0])


def _t_of(tr, k):
    return tr.rec['t'][k] if k < T else torch.zeros((tr.n, 1), device='cuda')


def test_recorder_runs_the_production_sampler(traj):
    rec, dyn = traj.rec, traj.ddpm.dynamics
    assert dyn.math_mode == 15 and dyn.deterministic_active     # 3xFP16 at H=256 and H=128
    assert rec['step'] == list(range(T - 1, -1, -1)) and len(rec['z']) == T + 1
    for i, (a, b) in enumerate(zip(rec['out'], traj.plain)):
        assert torch.equal(a, b), f'{traj.name}: output {i} of the recorded run differs from an unmodified call'
    assert torch.isfinite(rec['z'][T]).all() and torch.isfinite(rec['pocket'][T]).all()


def test_step_tables_every_step(traj):
    ddpm, rec, n = traj.ddpm, traj.rec, traj.n
    if traj.joint:
        t_table, coef_table = ddpm._joint_tables(T, 1, 'cuda')
    else:
        t_table, coef_table = ddpm._schedule_tables(T, T, 'cuda')
    target = rec['z'][0]
    for k, s in enumerate(rec['step']):
        # the eager loop's own t and s (sample_given_pocket / sample)
        s_array = torch.full((n, 1), fill_value=s, device='cuda')
        t_array = (s_array + 1) / T
        s_array = s_array / T
        assert torch.equal(rec['t'][k], t_array), f'{traj.name} step s={s}: t {float(rec["t"][k][0])}'
        # torch divides a CUDA tensor by a scalar as a multiplication by the rounded reciprocal, so t is within two ulp
        # of (s+1)/T rather than correctly rounded (0.996 and 0.99 come out one ulp high); the schedule looks gamma up at
        # round(t T), which must be s+1
        assert abs(float(rec['t'][k][0]) - (s + 1) / T) <= 2 * ulp32((s + 1) / T)
        assert torch.equal(torch.round(rec['t'][k] * T).long(), torch.full_like(s_array, s + 1, dtype=torch.long))
        if traj.joint:
            want = joint_step_coefficients(ddpm, s_array, t_array, target)
        else:
            want = torch.cat(ddpm._step_coefficients(ddpm.gamma(s_array), ddpm.gamma(t_array), target), 1)
        assert torch.equal(rec['coef3'][k], want), \
            f'{traj.name} step s={s}: coefficients {rec["coef3"][k][0].tolist()} vs eager {want[0].tolist()}'
        assert torch.equal(t_table[s], t_array[0]) and torch.equal(coef_table[s, :3], want[0])


def test_fused_update_every_step(traj):
    ddpm, rec, lm, pm = traj.ddpm, traj.rec, traj.lm, traj.pm
    dyn = ddpm.dynamics
    for k, s in enumerate(rec['step']):
        z, p, noise, coef3 = rec['z'][k], rec['pocket'][k], rec['noise'][k], rec['coef3'][k]
        with torch.no_grad():
            eps_l, eps_p = dyn(z, p, rec['t'][k], lm, pm)
        if traj.joint:
            got = joint_update(ddpm, z, p, eps_l, eps_p, noise, coef3, lm, pm)
            ref = lambda dt: joint_update_ref(z, p, eps_l, eps_p, noise, coef3, lm, pm, dt)
        else:
            got = ligand_update(ddpm, z, eps_l, noise, coef3, p, lm, pm)
            ref = lambda dt: ligand_update_ref(z, eps_l, noise, coef3, p, lm, pm, dt)
        assert torch.equal(got[0], rec['z'][k + 1]) and torch.equal(got[1], rec['pocket'][k + 1]), \
            f'{traj.name} step s={s}: eager denoiser + fused update differs from the graph replay'
        w32, w64 = ref(torch.float32), ref(torch.float64)
        assert_fp64_bound(rec['z'][k + 1], w32[0], w64[0], f'{traj.name} step s={s} ligand')
        assert_fp64_bound(rec['pocket'][k + 1], w32[1], w64[1], f'{traj.name} step s={s} pocket')


def _nets(tr):
    out = {}
    for label, mode, det in MODES:
        net = EGNNDynamics.from_config(tr.cfg, device='cuda')
        net.load_state_dict(tr.sd)
        net.eval()
        net.math_mode = mode
        net.deterministic = det
        out[label] = net
    return out


def _group(k):
    return 'early' if k < 8 else ('late' if k >= T - 8 else 'middle')


def test_denoiser_against_fp64_selected_steps(traj):
    tr, rec, lm, pm = traj, traj.rec, traj.lm, traj.pm
    nets = _nets(tr)
    rows, failures = [], []
    exempt = 0
    t0 = time.time()
    for k in SELECTED:
        z, p, t = rec['z'][k], rec['pocket'][k], _t_of(tr, k)
        edges = nets['3xfp16'].get_edges(lm, pm, z[:, :3], p[:, :3])
        o64 = egnn_oracle.denoiser_forward(tr.cfg, tr.sd, z, p, t, lm, pm, dtype=torch.float64, device='cuda', edges=edges)
        o32 = egnn_oracle.denoiser_forward(tr.cfg, tr.sd, z, p, t, lm, pm, device='cuda', edges=edges)
        vel32, h32 = column_errors(o32, o64)
        xmax = float(torch.cat((z[:, :3], p[:, :3])).abs().max())
        velmax = max(float(o[:, :3].abs().max()) for o in o64)
        # the project tolerance is asserted on the column groups where the fp32 oracle's own error leaves it the headroom it
        # was set with (the fp32 oracle within a tenth of it); see the module docstring
        held = [(side, cols) for side in (0, 1) for cols in (slice(0, 3), slice(3, None))
                if _within_tolerance(o32[side][:, cols], o64[side][:, cols], ATOL / 10, RTOL / 10)]
        exempt += 4 - len(held)
        row = dict(k=k, s=T - 1 - k, E=edges.shape[1], vel32=vel32, h32=h32, xmax=xmax, velmax=velmax, held=len(held))
        for label, net in nets.items():
            with torch.no_grad():
                got = net(z, p, t, lm, pm)
            torch.cuda.synchronize()
            what = f'{tr.name} k={k} (s={T - 1 - k}) {label}'
            if net.last_num_edges != edges.shape[1]:
                failures.append(f'{what}: forward used {net.last_num_edges} edges, get_edges {edges.shape[1]}')
            for side, cols in held:
                try:
                    assert_close(got[side][:, cols], o64[side][:, cols],
                                 f'{what} {("ligand", "pocket")[side]} {"vel" if cols.start == 0 else "h"} vs fp64')
                except AssertionError as e:
                    failures.append(str(e))
            vel, h = column_errors(got, o64)
            row[label] = (vel / vel32, h / h32)
            if vel > K * vel32 + FLOOR:
                failures.append(f'{what}: vel error {vel:.2e} > {K} x fp32 oracle error {vel32:.2e}')
            if h > K * h32 + FLOOR:
                failures.append(f'{what}: h error {h:.2e} > {K} x fp32 oracle error {h32:.2e}')
        rows.append(row)
    labels = [m[0] for m in MODES]
    print(f'\n[{tr.name}] denoiser vs fp64 at {len(SELECTED)} steps ({time.time() - t0:.1f} s): ratio err_native / '
          f'err_fp32_oracle, vel / h')
    print(f'{"k":>4} {"s":>4} {"E":>8} {"max|x|":>7} {"max|vel|":>8} {"tol":>3} {"fp32 oracle vel / h":>20}  '
          + '  '.join(f'{lb:>13}' for lb in labels))
    for r in rows:
        print(f'{r["k"]:>4} {r["s"]:>4} {r["E"]:>8} {r["xmax"]:>7.1f} {r["velmax"]:>8.2f} {r["held"]:>3} '
              f'{r["vel32"]:>9.2e} / {r["h32"]:.2e}  '
              + '  '.join(f'{r[lb][0]:>5.2f} / {r[lb][1]:<5.2f}' for lb in labels))
    for grp in ('early', 'middle', 'late'):
        sel = [r for r in rows if _group(r['k']) == grp]
        print(f'max {grp:>6} ({len(sel):>2} calls): ' + '  '.join(
            f'{lb} {max(r[lb][0] for r in sel):.2f} / {max(r[lb][1] for r in sel):.2f}' for lb in labels))
    print(f'column groups (ligand/pocket x vel/h) where the fp32 oracle misses a tenth of the project tolerance: {exempt} of '
          f'{4 * len(rows)}')
    assert not failures, '\n'.join(failures[:20])


def _within_tolerance(got, want, atol, rtol):
    err = (got.double() - want.double()).abs()
    return bool((err <= atol + rtol * want.double().abs()).all())


def test_edges_along_trajectory(traj):
    tr, rec, lm, pm = traj, traj.rec, traj.lm, traj.pm
    pairs = candidate_pairs(lm, pm)
    net = tr.ddpm.dynamics
    band = disagree = 0
    for k in range(T + 1):
        z, p = rec['z'][k], rec['pocket'][k]
        edges = net.get_edges(lm, pm, z[:, :3], p[:, :3])
        n, b, d, bad = compare_edges(tr.cfg, edges, z[:, :3], p[:, :3], lm, pm, pairs, DELTA_ULPS)
        assert not bad, f'{tr.name} k={k}: pairs outside the {DELTA_ULPS}-ulp band decided against float64: {bad}'
        band += b
        disagree += d
    print(f'\n[{tr.name}] edge lists at {T + 1} states, {pairs[0].numel()} same-graph pairs each: {band} pair-states within '
          f'{DELTA_ULPS} ulp of a cut-off, {disagree} of them decided differently from float64')


def test_planted_boundary_pairs():
    inp, meta = planted_batch()
    cfg = PLANT_CFG
    sd = syn.synthetic_state_dict(cfg, 0)
    net = EGNNDynamics.from_config(cfg, device='cuda')
    net.load_state_dict(sd)
    net.eval()
    xs = [x.cuda() for x in inp]
    edges = net.get_edges(xs[3], xs[4], xs[0][:, :3], xs[1][:, :3]).cpu()
    N = inp[0].shape[0] + inp[1].shape[0]
    keys = set((edges[0] * N + edges[1]).tolist())
    x = torch.cat((inp[0][:, :3], inp[1][:, :3])).double()
    in_band = 0
    for m in meta:
        i, j, cut, k = m['i'], m['j'], m['cut'], m['k']
        kept = i * N + j in keys
        what = f"{m['block']} {m['kind']} {k:+d} ulp (cut {cut})"
        assert kept == (j * N + i in keys), what
        d = float((x[i] - x[j]).pow(2).sum().sqrt())
        delta = DELTA_ULPS * ulp32(cut)
        if k == 0:
            assert kept, f'{what}: a pair exactly at the cut-off must be kept (d <= cut)'
        elif m['kind'] == 'axis':       # fp32 difference, square and sqrt are exact along an axis
            assert kept == (k < 0), f'{what}: d = {d!r}'
        elif d < cut - delta:
            assert kept, f'{what}: d = {d!r} is more than {DELTA_ULPS} ulp inside'
        elif d > cut + delta:
            assert not kept, f'{what}: d = {d!r} is more than {DELTA_ULPS} ulp outside'
        else:
            in_band += 1
    assert all(n * N + n in keys for n in range(N))            # self-pairs (d = 0)
    _, _, _, bad = compare_edges(cfg, edges, inp[0][:, :3], inp[1][:, :3], inp[3], inp[4])
    assert not bad
    with torch.no_grad():
        out = net(*xs)
    torch.cuda.synchronize()
    assert net.last_num_edges == edges.shape[1] == len(keys)
    o64 = egnn_oracle.denoiser_forward(cfg, sd, *inp, dtype=torch.float64, edges=edges)
    assert_close(out[0], o64[0], 'planted batch ligand vs fp64 on the native edges')
    assert_close(out[1], o64[1], 'planted batch pocket vs fp64 on the native edges')
    print(f'\nplanted pairs: {len(meta)}, generic pairs within {DELTA_ULPS} ulp of the cut-off (not asserted): {in_band}')
