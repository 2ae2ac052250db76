"""GPU: the RePaint inpainting samplers checked replay by replay along production schedules, and every seeded draw of those
runs against the Philox restatement.

The runs (tests/repaint_cases.py RUNS; T = 500, polynomial_2, synthetic weights, deterministic mode, 3xFP16, graph engine):
``inpaint_50x20`` (ConditionalDDPM.inpaint, configs[4]: 64 x (25 + 175) atoms, the first 10 of 25 fixed, center='ligand',
50 sub-sampled steps x 20 resamplings = 1000 replays), ``inpaint_500x1``, ``joint_jump`` (EnVariationalDiffusion.inpaint,
16 x (25 + 175), ligand and pocket partly fixed, resamplings=2, jump_length=10), ``joint_frames`` (4 graphs, jump_length=1,
resamplings=3, return_frames=5, timesteps=25: the eager jump between replays runs at s = 20, 15, 10, 5, 0) and
``diversify`` (noising_steps=100 right after a sample_given_pocket call, replaying its captured 'reverse' graph from
s = 99).  Each run is made unseeded and with seeds=; a Recorder (repaint_cases) wraps the sampler's graph getter so that
every replay of the production graphs is recorded.  Every check is teacher forced: kernel and reference get the same
recorded fp32 state.

* The recorded call gives the same bits as an unmodified call; replay kinds follow the schedule.
* Tables and counters, every replay: step and u as the eager loop walks them; t, coef3, coef4 bit for bit against the
  eager loop's torch ops for that (s, u) (the joint t_back included); sub-sampled: round(t T) = (s+1) T / timesteps.
* Fused iteration, every replay: the eager native denoiser + dsb_ddpm_ligand_update + dsb_ddpm_inpaint_update (or the
  joint pair) on the recorded input and noise reproduce the replay bit for bit, and meet ddpm_cases.assert_fp64_bound
  against the float64 eager RePaint ops, ligand and pocket.  Pocket h columns unchanged; after a re-noise or jump the
  ligand (joint: ligand+pocket) COM is zero, and otherwise the COM of the fixed nodes equals that of the denoised sample,
  within the same bound.  Eager jumps between replays are held to the same bound.
* Denoiser against float64 at selected replays (first 8, every 50th, last 8, the 20 resamplings at s = 0, the t = 0
  call) in 3xFP16, 3xTF32, fp32 (deterministic) and 3xFP16 default mode, with the criteria of test_gpu_trajectory.py.
* Edges, every replay: compare_edges against float64 distances outside the 4-ulp band.
* Seeded draws: every replay's draw ids are draw_id(STAGE_LOOP, s, u, purpose) for the purposes it draws; every noise
  buffer of graphs 0, 1, 37, 63 (all graphs of the joint runs), and every host-side draw, equals the numpy Philox
  restatement within 8 ulp of max(|z|, 1); no (draw id, role) repeats in a run; the run's id sequence is the schedule's,
  and the eager engine issues the same sequence; diversify's partial noising meets the float64 bound.

Measured ratios, pair-states in the 4-ulp band and the runtime: DESIGN.md §5.

Planted defects (each on a scratch copy, none committed) and the test that caught it:
1. ddpm_inpaint_kernel takes dx over all ligand atoms, not the fixed ones: test_fused_iteration_every_replay
   [inpaint_500x1], replay 0, ligand 1.1 from float64.
2. The known part no longer follows the pocket COM (shift dropped): test_fused_iteration_every_replay[inpaint_500x1],
   replay 0, pocket 3e-2 from float64.
3. The re-noise COM sum takes only the first 128 elements of the block's strided loop:
   test_fused_iteration_every_replay[inpaint_50x20], replay 0, ligand 0.52 from float64.
4. inpaint_renoise also does step -= 1: test_tables_and_counters_every_replay[inpaint_50x20] (step counter).
5. u not advanced on re-noise, in both engines: test_repaint_cases_cpu.py::test_schedule_matches_eager_draws
   [inpaint_50x20].  On the GPU the seeded 50 x 20 run fails before its checks: the same re-noise drawn 20 times per
   step makes the chain diverge (NaN status).
6. PURPOSE_KNOWN and PURPOSE_RENOISE swapped in the graph engine only: test_seeded_draws[inpaint_50x20-seeded] (the
   noise buffers do not restate their purposes' ids).
7. The joint t_back clamp off by one (max = timesteps - 1): test_tables_and_counters_every_replay[joint_frames] (coef4)
   and test_repaint_cases_cpu.py::test_joint_tables_clamp_t_back.
8. ddpm_joint_inpaint_kernel's jump uses the known-part noise (nx1, nhl1, nhp1) where the jump noise belongs:
   test_fused_iteration_every_replay[joint_frames], replay 1, ligand 4.1 from float64.  Substituting only the
   per-graph mean n1 for n3 is not a defect of the output: it shifts every node of a graph by one constant, which
   the joint COM removal that follows cancels.
"""
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import repaint_cases as rc
from ddpm_cases import assert_fp64_bound
from helpers import ATOL, RTOL, assert_close
from stress_cases import column_errors
from trajectory_cases import T, candidate_pairs, compare_edges, ligand_update, ligand_update_ref, joint_update, \
    joint_update_ref, make_ddpm
from diffsbdd_b200 import _native, seeded, synthetic as syn
from diffsbdd_b200.config import FULLATOM_COND, FULLATOM_JOINT
from diffsbdd_b200.dynamics import EGNNDynamics
from diffsbdd_b200.en_diffusion import scatter_mean
from oracle import egnn_oracle

pytestmark = pytest.mark.gpu

K = 10.0
FLOOR = 1e-7
DELTA_ULPS = 4
CHECKED_GRAPHS = (0, 1, 37, 63)
MODES = [('3xfp16', '3xfp16', True), ('3xtf32', '3xtf32', True), ('fp32', 'fp32', True), ('3xfp16 dflt', '3xfp16', False)]
EAGER_RUNS = ('inpaint_50x20', 'joint_jump')


@pytest.fixture(scope='module', autouse=True)
def no_tf32():
    prev = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev


@pytest.fixture(scope='module')
def models():
    return {False: make_ddpm(FULLATOM_COND, False), True: make_ddpm(FULLATOM_JOINT, True)}


def _recorded_and_plain(ddpm, name, joint, seeds):
    if name == 'diversify':
        rc.sample_before_diversify(ddpm, seeds)
        cached = next(iter(ddpm._graph_cache.values()))['graphs']['reverse']
    with rc.Recorder(ddpm, joint) as rec:
        rec.out = rc.call(ddpm, name, seeds)
    plain = rc.call(ddpm, name, seeds)
    rec.cached = cached if name == 'diversify' else None
    return rec, plain


@pytest.fixture(scope='module', params=[(n, s) for n in rc.RUNS for s in (False, True)],
            ids=lambda p: p[0] + ('-seeded' if p[1] else ''))
def run(request, models):
    name, is_seeded = request.param
    spec = rc.RUNS[name]
    joint = spec['joint']
    ddpm = models[joint]
    seeds = rc.run_seeds(spec['n']) if is_seeded else None
    t0 = time.time()
    rec, plain = _recorded_and_plain(ddpm, name, joint, seeds)
    eager = None
    if is_seeded and name in EAGER_RUNS:
        ddpm.loop_engine = 'eager'
        try:
            with rc.Recorder(ddpm, joint) as eager:
                rc.call(ddpm, name, seeds)
        finally:
            ddpm.loop_engine = 'auto'
    torch.cuda.synchronize()
    print(f'\n[{name}{" seeded" if is_seeded else ""}] recorded + unmodified runs: {time.time() - t0:.1f} s, '
          f'{len(rec.replays)} replays')
    ctx = rec.ctx
    yield SimpleNamespace(name=name, spec=spec, joint=joint, seeded=is_seeded, seeds=seeds, ddpm=ddpm, rec=rec,
                          plain=plain, eager=eager, sched=rc.schedule_of(name), lm=ctx['lm'], pm=ctx['pm'],
                          cfg=FULLATOM_JOINT if joint else FULLATOM_COND,
                          timesteps=spec.get('timesteps', T), n=spec['n'])


def _state(run, k, which='in'):
    """(ligand, pocket) on the device before (``in``) or after (``out``) replay k."""
    r = run.rec.replays[k]
    z, p = (r['z'], r['p']) if which == 'in' else (r['out_z'], r['out_p'])
    z, p = z.cuda(), p.cuda()
    if not run.joint:
        p = torch.cat((p, run.rec.ctx['h0']), 1)
    return z, p


def test_recorded_call_is_the_production_call(run):
    rec = run.rec
    assert run.ddpm.dynamics.math_mode == 15 and run.ddpm.dynamics.deterministic_active
    for i, (a, b) in enumerate(zip(rec.out, run.plain)):
        assert torch.equal(a, b), f'{run.name}: output {i} of the recorded call differs from an unmodified call'
    assert [r['kind'] for r in rec.replays] == [e.kind for e in run.sched]
    eager_jumps = [k for k, e in enumerate(run.sched) if e.eager_jump]
    assert sorted(rec.jumps) == eager_jumps
    if run.name == 'joint_frames':
        assert len(eager_jumps) == 5
    if run.name == 'diversify':          # the capture of sample_given_pocket, replayed from s = 99
        assert all(r['graph'] is rec.cached for r in rec.replays) and rec.replays[0]['step'] == 99
    assert all(torch.isfinite(r['out_z']).all() for r in rec.replays)


def test_tables_and_counters_every_replay(run):
    ddpm, rec, n, ts = run.ddpm, run.rec, run.n, run.timesteps
    jump = run.spec.get('jump_length', 1)
    for k, (r, e) in enumerate(zip(rec.replays, run.sched)):
        what = f'{run.name} replay {k} ({e.kind}, s={e.s}, u={e.u})'
        assert r['step'] == e.s, f'{what}: step counter {r["step"]}'
        if run.seeded:
            assert r['u'] == e.u, f'{what}: u counter {r["u"]}'
        t, coef3, coef4 = (x.cpu() for x in rc.eager_coefficients(ddpm, run.joint, e.s, ts, n, 'cuda', jump))
        assert torch.equal(r['t'], t), f'{what}: t {float(r["t"][0])}'
        assert torch.equal(torch.round(r['t'] * T).long(), torch.full((n, 1), (e.s + 1) * T // ts)), what
        assert torch.equal(r['coef3'], coef3), f'{what}: reverse coefficients {r["coef3"][0].tolist()} vs {coef3[0].tolist()}'
        if e.kind != 'reverse':
            assert torch.equal(r['coef4'], coef4), f'{what}: RePaint coefficients {r["coef4"][0].tolist()} vs {coef4[0].tolist()}'


def _com(x, mask, sel=None):
    x, mask = x.double(), mask
    if sel is not None:
        x, mask = x[sel], mask[sel]
    return scatter_mean(x, mask)


def _assert_com_bound(got, want32, want64, scale, what):
    """|got - want64| within max(2 |want32 - want64|, 4 ulp(scale)): the fp64 bound on a COM of coordinates of magnitude
    up to ``scale``."""
    err = float((got - want64).abs().max())
    err32 = float((want32 - want64).abs().max())
    bound = max(2.0 * err32, 4.0 * rc.ulp_of(scale))
    assert err <= bound, f'{what}: {err:.3e} > {bound:.3e} (fp32 torch ops {err32:.3e})'


def test_fused_iteration_every_replay(run):
    ddpm, rec, lm, pm = run.ddpm, run.rec, run.lm, run.pm
    dyn, ctx = ddpm.dynamics, rec.ctx
    cuda = lambda xs: tuple(x.cuda() for x in xs)
    for k, (r, e) in enumerate(zip(rec.replays, run.sched)):
        what = f'{run.name} replay {k} ({e.kind}, s={e.s}, u={e.u})'
        z, p = _state(run, k)
        out_z, out_p = _state(run, k, 'out')
        t, coef3, coef4 = r['t'].cuda(), r['coef3'].cuda(), r['coef4'].cuda()
        with torch.no_grad():
            eps_l, eps_p = dyn(z, p, t, lm, pm)
        if run.joint:
            kn = ctx['known']
            n_rev, n1 = cuda(r['n_rev']), cuda(r['n_known'])
            n3 = cuda(r['n_jump']) if e.kind == 'inpaint_jump' else None
            zd, pd = joint_update(ddpm, z, p, eps_l, eps_p, n_rev, coef3, lm, pm)
            got = rc.joint_inpaint_update(ddpm, zd, pd, kn, n1, n3, coef4, lm, pm)

            def ref(dt):
                wl, wp = joint_update_ref(z, p, eps_l, eps_p, n_rev, coef3, lm, pm, dt)
                return (wl, wp) + rc.joint_inpaint_update_ref(wl, wp, kn['xl'], kn['xp'], kn['fl'], kn['fp'], n1, n3, coef4,
                                                              lm, pm, dt)
            sel_l, sel_p = kn['fl'].bool(), kn['fp'].bool()
        else:
            noise = r['noise'].cuda()
            zd, pd = ligand_update(ddpm, z, eps_l, noise, coef3, p, lm, pm)
            n1 = r['noise1'].cuda() if e.kind != 'reverse' else None
            n2 = r['noise2'].cuda() if e.kind == 'inpaint_renoise' else None
            ip = ctx.get('inpaint')
            got = (zd, pd) if e.kind == 'reverse' else \
                rc.inpaint_update(ddpm, zd, pd, ip['known'], ip['com0'], ip['fixed'], n1, n2, coef4, lm, pm)

            def ref(dt):
                wz, wp = ligand_update_ref(z, eps_l, noise, coef3, p, lm, pm, dt)
                if e.kind == 'reverse':
                    return wz, wp, wz, wp
                return (wz, wp) + rc.inpaint_update_ref(wz, wp, ip['known'], ip['com0'], ip['fixed'], n1, n2, coef4, lm, pm, dt)
            assert r['h_same'], f'{what}: pocket h columns changed'
            sel_l = ip['fixed'].bool() if ip is not None else None
        assert torch.equal(got[0], out_z) and torch.equal(got[1], out_p), \
            f'{what}: eager denoiser + fused kernels differ from the graph replay'
        w32, w64 = ref(torch.float32), ref(torch.float64)
        assert_fp64_bound(out_z, w32[2], w64[2], f'{what} ligand')
        assert_fp64_bound(out_p[:, :3] if not run.joint else out_p, (w32[3] if run.joint else w32[3][:, :3]),
                          (w64[3] if run.joint else w64[3][:, :3]), f'{what} pocket')
        scale = float(torch.cat((out_z[:, :3], out_p[:, :3])).abs().max())
        renoised = e.kind in ('inpaint_renoise', 'inpaint_jump')
        if e.kind == 'reverse':
            continue
        if run.joint:
            x = lambda a, b: torch.cat((a[:, :3], b[:, :3]))
            cm, sel = torch.cat((lm, pm)), torch.cat((sel_l, sel_p))
            if renoised:             # joint COM zero after the jump back
                _assert_com_bound(_com(x(out_z, out_p), cm), _com(x(w32[2], w32[3]), cm), _com(x(w64[2], w64[3]), cm),
                                  scale, f'{what} joint COM')
            else:                    # COM of the fixed nodes = that of the denoised sample
                d = lambda a, b, c, f: _com(x(a, b), cm, sel) - _com(x(c, f), cm, sel)
                _assert_com_bound(d(out_z, out_p, zd, pd), d(w32[2], w32[3], w32[0], w32[1]), d(w64[2], w64[3], w64[0], w64[1]),
                                  scale, f'{what} fixed-node COM')
        else:
            if renoised:
                _assert_com_bound(_com(out_z[:, :3], lm), _com(w32[2][:, :3], lm), _com(w64[2][:, :3], lm), scale,
                                  f'{what} ligand COM')
            else:
                d = lambda a, b: _com(a[:, :3], lm, sel_l) - _com(b[:, :3], lm, sel_l)
                _assert_com_bound(d(out_z, zd), d(w32[2], w32[0]), d(w64[2], w64[0]), scale, f'{what} fixed-atom COM')
        if k in rec.jumps:
            _check_eager_jump(run, k)


def _check_eager_jump(run, k):
    """The eager jump back after replay k: its input is the replay's output, the next replay starts from its output, and
    the output meets the fp64 bound on the recorded input and noise."""
    j, rec, lm, pm = run.rec.jumps[k], run.rec, run.lm, run.pm
    what = f'{run.name} eager jump after replay {k}'
    assert torch.equal(j['zl'], rec.replays[k]['out_z']) and torch.equal(j['zp'], rec.replays[k]['out_p']), what
    if k + 1 < len(rec.replays):
        assert torch.equal(rec.replays[k + 1]['z'], j['out'][0]) and torch.equal(rec.replays[k + 1]['p'], j['out'][1]), what
    args = [x.cuda() for x in (j['zl'], j['zp'], j['eps'][0], j['eps'][1], j['gamma_t'], j['gamma_s'])]
    w32 = rc.joint_jump_ref(run.ddpm, *args, lm, pm, torch.float32)
    w64 = rc.joint_jump_ref(run.ddpm, *args, lm, pm, torch.float64)
    assert_fp64_bound(j['out'][0], w32[0], w64[0], f'{what} ligand')
    assert_fp64_bound(j['out'][1], w32[1], w64[1], f'{what} pocket')


def _selected(run):
    n = len(run.rec.replays)
    sel = set(range(min(8, n))) | set(range(50, n - 8, 50)) | set(range(max(0, n - 8), n))
    if run.name == 'inpaint_50x20':
        sel |= {k for k, e in enumerate(run.sched) if e.s == 0}
    return sorted(sel) + [n]                                   # n: the t = 0 call


def _nets(cfg):
    sd = syn.synthetic_state_dict(cfg, 0)
    out = {}
    for label, mode, det in MODES:
        net = EGNNDynamics.from_config(cfg, device='cuda')
        net.load_state_dict(sd)
        net.eval()
        net.math_mode = mode
        net.deterministic = det
        out[label] = net
    return sd, out


def _group(k, n):
    return 'early' if k < 8 else ('late' if k >= n - 8 else 'middle')


def test_denoiser_against_fp64_selected_replays(run):
    if run.seeded:
        pytest.skip('checked on the unseeded run of the same schedule')
    rec, lm, pm, cfg = run.rec, run.lm, run.pm, run.cfg
    sd, nets = _nets(cfg)
    n = len(rec.replays)
    rows, failures = [], []
    t0 = time.time()
    for k in _selected(run):
        if k < n:
            z, p = _state(run, k)
            t = rec.replays[k]['t'].cuda()
        else:
            z, p = _state(run, n - 1, 'out')
            t = torch.zeros((run.n, 1), device='cuda')
        edges = nets['3xfp16'].get_edges(lm, pm, z[:, :3], p[:, :3])
        o64 = egnn_oracle.denoiser_forward(cfg, sd, z, p, t, lm, pm, dtype=torch.float64, device='cuda', edges=edges)
        o32 = egnn_oracle.denoiser_forward(cfg, sd, z, p, t, lm, pm, device='cuda', edges=edges)
        vel32, h32 = column_errors(o32, o64)
        held = [(side, cols) for side in (0, 1) for cols in (slice(0, 3), slice(3, None))
                if _within_tolerance(o32[side][:, cols], o64[side][:, cols], ATOL / 10, RTOL / 10)]
        row = dict(k=k, E=edges.shape[1], vel32=vel32, h32=h32)
        for label, net in nets.items():
            with torch.no_grad():
                got = net(z, p, t, lm, pm)
            torch.cuda.synchronize()
            what = f'{run.name} replay {k} {label}'
            if net.last_num_edges != edges.shape[1]:
                failures.append(f'{what}: forward used {net.last_num_edges} edges, get_edges {edges.shape[1]}')
            for side, cols in held:
                try:
                    assert_close(got[side][:, cols], o64[side][:, cols], f'{what} side {side} cols {cols.start} vs fp64')
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
    print(f'\n[{run.name}] denoiser vs fp64 at {len(rows)} calls ({time.time() - t0:.1f} s): ratio err_native / '
          f'err_fp32_oracle, vel / h')
    for grp in ('early', 'middle', 'late'):
        sel = [r for r in rows if _group(r['k'], n + 1) == grp]
        if sel:
            print(f'max {grp:>6} ({len(sel):>2} calls): ' + '  '.join(
                f'{lb} {max(r[lb][0] for r in sel):.2f} / {max(r[lb][1] for r in sel):.2f}' for lb in labels))
    assert not failures, '\n'.join(failures[:20])


def _within_tolerance(got, want, atol, rtol):
    err = (got.double() - want.double()).abs()
    return bool((err <= atol + rtol * want.double().abs()).all())


def test_edges_every_replay(run):
    rec, lm, pm = run.rec, run.lm, run.pm
    pairs = candidate_pairs(lm, pm)
    net = run.ddpm.dynamics
    band = disagree = 0
    n = len(rec.replays)
    for k in range(n + 1):
        z, p = _state(run, k) if k < n else _state(run, n - 1, 'out')
        edges = net.get_edges(lm, pm, z[:, :3], p[:, :3])
        _, b, d, bad = compare_edges(run.cfg, edges, z[:, :3], p[:, :3], lm, pm, pairs, DELTA_ULPS)
        assert not bad, f'{run.name} replay {k}: pairs outside the {DELTA_ULPS}-ulp band decided against float64: {bad}'
        band += b
        disagree += d
    print(f'\n[{run.name}] edge lists at {n + 1} states, {pairs[0].numel()} same-graph pairs each: {band} pair-states within '
          f'{DELTA_ULPS} ulp of a cut-off, {disagree} of them decided differently from float64')


def _rows_of(mask, graphs):
    return torch.isin(mask.cpu(), torch.tensor(graphs))


def test_seeded_draws(run):
    if not run.seeded:
        pytest.skip('unseeded run: torch generator')
    rec, lm, pm = run.rec, run.lm.cpu(), run.pm.cpu()
    seeds = np.array(run.seeds, dtype=np.uint64)
    graphs = list(range(run.n)) if run.joint else list(CHECKED_GRAPHS)
    sl, sp = _rows_of(lm, graphs), _rows_of(pm, graphs)
    lm_s, pm_s = lm[sl].numpy(), pm[sp].numpy()
    A, R = run.ddpm.atom_nf, run.ddpm.residue_nf
    n_checked = 0

    def check(buf, role, draw, what):
        nonlocal n_checked
        if role == _native.RNG_LIGAND:
            got = buf[sl]
        elif role == _native.RNG_POCKET:
            got = buf[sp]
        else:
            got = buf[torch.cat((sl, sp))]
        rc.assert_restated(got, role, buf.shape[1], seeds, draw, lm_s, pm_s, what)
        n_checked += 1

    for k, (r, e) in enumerate(zip(rec.replays, run.sched)):
        what = f'{run.name} replay {k} ({e.kind}, s={e.s}, u={e.u})'
        for p in e.purposes:
            want = seeded.draw_id(seeded.STAGE_LOOP, e.s, e.u, p)
            assert int(r['draw'][p]) == want, f'{what}: purpose {p} drew {rc.decode(r["draw"][p])}, want {rc.decode(want)}'
        if run.joint:
            bufs = {rc.REV: r['n_rev'], rc.KNOWN: r['n_known']}
            if e.kind == 'inpaint_jump':
                bufs[rc.RENOISE] = r['n_jump']
            for p, triple in bufs.items():
                for buf, role in zip(triple, rc.JOINT_ROLES):
                    check(buf, role, int(r['draw'][p]), f'{what} purpose {p} role {role}')
        else:
            bufs = {rc.REV: r['noise'], rc.KNOWN: r.get('noise1'), rc.RENOISE: r.get('noise2')}
            for p in e.purposes:
                check(bufs[p], _native.RNG_LIGAND, int(r['draw'][p]), f'{what} purpose {p}')
    for draw, by_role in rec.fills.items():                     # prior, partial noising, final, eager jumps
        for role, buf in by_role.items():
            check(buf, role, draw, f'{run.name} host draw {rc.decode(draw)} role {role}')
    assert len(set(rec.draws)) == len(rec.draws), f'{run.name}: a (draw id, role) repeats within the run'
    assert rec.draws == rc.draw_sequence(run.name), f'{run.name}: draw sequence differs from the schedule'
    if run.eager is not None:
        assert run.eager.draws == rec.draws, f'{run.name}: the eager engine issues another draw sequence'
    print(f'\n[{run.name}] {len(rec.draws)} seeded draws in sequence, {n_checked} noise buffers restated')


def test_partial_noising(run):
    if run.name != 'diversify':
        pytest.skip('diversify only')
    rec, ddpm = run.rec, run.ddpm
    inp, (z, p, eps) = rec.partial['inp'], rec.partial['out']
    lm, pm = inp['lm'], inp['pm']
    n = int(lm.max()) + 1
    t = torch.ones(size=(n, 1), device='cuda').float() * inp['noising_steps'] / T      # partially_noised_ligand's t
    gamma = ddpm.gamma(t)

    def ref(dt):
        xl = torch.cat((inp['x'], inp['one_hot']), 1).to(dt)
        xp = torch.cat((inp['px'], inp['ph']), 1).to(dt)
        mean = scatter_mean(xl[:, :3], lm)
        xl[:, :3] -= mean[lm]
        xp[:, :3] -= mean[pm]
        g = gamma.to(dt)
        alpha, sigma = ddpm.alpha(g, xl), ddpm.sigma(g, xl)
        zl = alpha[lm] * xl + sigma[lm] * eps.to(dt)
        m2 = scatter_mean(zl[:, :3], lm)
        zl[:, :3] -= m2[lm]
        xp[:, :3] -= m2[pm]
        return zl, xp
    w32, w64 = ref(torch.float32), ref(torch.float64)
    assert_fp64_bound(z, w32[0], w64[0], 'partial noising ligand')
    assert_fp64_bound(p, w32[1], w64[1], 'partial noising pocket')
    assert rec.replays[0]['z'].equal(z.cpu()) and rec.replays[0]['p'].equal(p[:, :3].cpu())
    if run.seeded:
        draw = seeded.draw_id(seeded.STAGE_PARTIAL)
        assert torch.equal(rec.fills[draw][_native.RNG_LIGAND], eps.cpu())
