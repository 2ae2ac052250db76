"""GPU: few-step RePaint inpainting and diversify (DESIGN §14).

1. dsb_ddpm_multistep_inpaint_update against float64 (fast_repaint_cases) on every output (z, pocket, history), both models,
   committing or not, with and without re-noise, on a first (w = 0) and a later step: configs[2] and a ragged batch with an
   empty pocket, a one-atom ligand, a graph with every atom fixed and one with none fixed.
2. The graph engine teacher-forced against float64 replay by replay along seeded runs: the captured rounds are recorded (the
   graph getter is wrapped, so a recorded call gives the bits of an unmodified one) and each is restated on its own recorded
   input, with the denoiser output recomputed on that input (deterministic mode: the same bits).  bench's inpaint shape at
   N = 50 with 1 and 3 resamplings, the joint production model with its pocket fixed, and diversify from 100 noising steps.
3. Seeded, deterministic runs, both engines, both models: graphs 0, 37, 63 alone and in a reversed sub-batch equal the full
   batch in every frame.
4. A sampler switch re-captures and switching back repeats the bits; diversify with another noising_steps uses its own table;
   sampler='ddpm' is the default call; a NaN reports as it does for the ancestral sampler.
"""
import ctypes as C

import pytest
import torch

from ddpm_cases import HIST, JOINT_CFG, assert_fp64_bound
from fast_repaint_cases import cond_round_ref, joint_round_ref
from fast_sampler_cases import ddim_ref, multistep_ref
from trajectory_cases import COND_LIG, COND_POC, JOINT_LIG, JOINT_POC, make_ddpm
from diffsbdd_b200 import _native, seeded, synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM
from diffsbdd_b200.config import FULLATOM_COND, FULLATOM_JOINT
from diffsbdd_b200.distributed import shard_pocket
from diffsbdd_b200.dynamics import EGNNDynamics
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion

pytestmark = pytest.mark.gpu
N = 50
RUNS = [('ddim', 0.0), ('ddim', 0.5), ('ddim', 1.0), ('dpmpp_2m', 0.0)]


# ---- 1. the kernel ------------------------------------------------------------------------------------------------------
SHAPES = {'configs2': ([25] * 64, [175] * 64), 'ragged': ([7, 1, 12, 3, 9], [30, 0, 9, 140, 11])}


def _kernel(joint, bufs, coef, lm, pm, A, R, renoise, commit):
    """dsb_ddpm_multistep_inpaint_update on copies of the state; returns (z_lig, z_pocket, hist_lig[, hist_pocket])."""
    zl, zp, hl, hp = (x.clone() for x in (bufs['zl'], bufs['zp'], bufs['hl'], bufs['hp']))
    P = lambda x: None if x is None else x.data_ptr()
    b = bufs
    if joint:
        n1, n3 = b['nk'], (b['nr'] if renoise else (None, None, None))
        extra = (P(zl), P(zp), P(hl), P(hp), P(b['el']), P(b['ep']), P(b['xl']), P(b['xp']), None, P(b['fl']), P(b['fp']),
                 *[P(x) for x in n1], *[P(x) for x in n3])
    else:
        extra = (P(zl), P(zp), P(hl), None, P(b['el']), None, P(b['xl']), None, P(b['com0']), P(b['fl']), None,
                 P(b['nkc']), None, None, P(b['nrc']) if renoise else None, None, None)
    _native.check(_native.load().dsb_ddpm_multistep_inpaint_update(
        *extra, P(coef), P(lm), P(pm), zl.shape[0], zp.shape[0], coef.shape[0], A, R, int(joint), int(commit),
        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return (zl, zp, hl, hp) if joint else (zl, zp, hl)


def _refs(joint, b, coef, lm, pm, renoise, commit):
    cf, cr = coef[:, :5], coef[:, 5:]
    if joint:
        args = (b['zl'], b['zp'], b['hl'], b['hp'], b['el'], b['ep'], None, b['nk'], b['nr'] if renoise else None, cf, cr,
                b['xl'], b['xp'], b['fl'], b['fp'], lm, pm, 'dpmpp_2m', commit)
        return [joint_round_ref(*args, d) for d in (torch.float32, torch.float64)]
    args = (b['zl'], b['zp'], b['hl'], b['el'], None, b['nkc'], b['nrc'] if renoise else None, cf, cr, b['xl'], b['com0'],
            b['fl'], lm, pm, 'dpmpp_2m', commit)
    return [cond_round_ref(*args, d) for d in (torch.float32, torch.float64)]


@pytest.mark.parametrize('step', ['first', 'later'])
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('joint', [False, True], ids=['cond', 'joint'])
def test_multistep_inpaint_kernel_against_float64(joint, shape, step):
    cfg = FULLATOM_JOINT if joint else FULLATOM_COND
    A, R = cfg.atom_nf, cfg.residue_nf
    n_lig, n_poc = SHAPES[shape]
    n = len(n_lig)
    g = torch.Generator(device='cuda').manual_seed(8)
    dev = 'cuda'
    lm = torch.repeat_interleave(torch.arange(n, device=dev), torch.tensor(n_lig, device=dev))
    pm = torch.repeat_interleave(torch.arange(n, device=dev), torch.tensor(n_poc, device=dev))
    rnd = lambda r, c, s=1.0: torch.randn((r, c), device=dev, generator=g) * s
    NL, NP = len(lm), len(pm)
    fl = (torch.rand(NL, device=dev, generator=g) < 0.4).float()
    fp = (torch.rand(NP, device=dev, generator=g) < 0.7).float()
    if shape == 'ragged':                       # graph 2: every node fixed; graph 4: none
        fl[lm == 2], fp[pm == 2], fl[lm == 4], fp[pm == 4] = 1., 1., 0., 0.
    b = dict(zl=rnd(NL, 3 + A), zp=rnd(NP, 3 + R, 4.0), hl=rnd(NL, 3 + A, 2.0), hp=rnd(NP, 3 + R, 2.0), el=rnd(NL, 3 + A),
             ep=rnd(NP, 3 + R), xl=rnd(NL, 3 + A, 1.5), xp=rnd(NP, 3 + R, 3.0), com0=rnd(n, 3), fl=fl, fp=fp,
             nk=(rnd(NL + NP, 3), rnd(NL, A), rnd(NP, R)), nr=(rnd(NL + NP, 3), rnd(NL, A), rnd(NP, R)),
             nkc=rnd(NL, 3 + A), nrc=rnd(NL, 3 + A))
    ddpm = make_ddpm(FULLATOM_COND.with_(n_layers=1), False, timesteps=500)
    _, fast = ddpm._fast_tables(N, 'dpmpp_2m', 0.0, 'cuda')
    _, anc = ddpm._schedule_tables(N, N, 'cuda')
    table = torch.cat((fast, anc[:, 3:]), 1)
    rows = torch.tensor([N - 1 if step == 'first' else 20, 30, 5, 44, 12], device=dev)
    coef = table[rows[torch.arange(n, device=dev) % 5]].contiguous()
    if step == 'first':
        coef[:, 4] = 0
    for renoise in (False, True):
        for commit in (False, True):
            got = _kernel(joint, b, coef, lm, pm, A, R, renoise, commit)
            refs = _refs(joint, b, coef, lm, pm, renoise, commit)
            what = f'{shape} {step} renoise={renoise} commit={commit}'
            for k, name in enumerate(('z_lig', 'z_pocket', 'hist_lig', 'hist_pocket')[:len(got)]):
                assert torch.isfinite(got[k]).all(), f'{what} {name}'
                assert_fp64_bound(got[k], refs[0][k], refs[1][k], f'{what} {name}')
            if not joint:
                assert torch.equal(got[1][:, 3:], b['zp'][:, 3:]), 'the conditional pocket features must not change'
            if not commit:
                assert torch.equal(got[2][:, 3:], b['hl'][:, 3:]), 'a round that does not commit only translates the history'
            again = _kernel(joint, b, coef, lm, pm, A, R, renoise, commit)
            assert all(torch.equal(x, y) for x, y in zip(got, again))
            # a graph's result does not depend on the rest of its batch: graph 1 alone
            l1, p1 = lm == 1, pm == 1
            sub = {k: (tuple(x[torch.cat((l1, p1))] if x.shape[0] == NL + NP else x[l1] if x.shape[0] == NL else x[p1]
                             for x in v) if isinstance(v, tuple) else
                       v[1:2] if k == 'com0' else v[l1] if v.shape[0] == NL else v[p1]) for k, v in b.items()}
            one = _kernel(joint, sub, coef[1:2].contiguous(), lm[l1] - 1, pm[p1] - 1, A, R, renoise, commit)
            assert torch.equal(one[0], got[0][l1]) and torch.equal(one[1], got[1][p1]) and torch.equal(one[2], got[2][l1])
    # a first step never reads the history
    if step == 'first':
        nan = dict(b, hl=torch.full_like(b['hl'], float('nan')), hp=torch.full_like(b['hp'], float('nan')))
        got = _kernel(joint, nan, coef, lm, pm, A, R, True, True)
        assert all(torch.isfinite(x).all() for x in got)


# ---- 2. the graph engine, teacher-forced --------------------------------------------------------------------------------
COND_KEYS = ('z', 'pocket', 'hist', 'noise', 'noise1', 'noise2', 't', 'coef_fast', 'coef4', 'coef9', 'step', 'u', 'draw')
JOINT_KEYS = ('zl', 'zp', 'hist', 'n_rev', 'n_known', 'n_jump', 't', 'coef_fast', 'coef4', 'coef9', 'step', 'u', 'draw')


def _snap(st, keys):
    out = {}
    for k in keys:
        if k in st:
            v = st[k]
            out[k] = tuple(x.clone() for x in v) if isinstance(v, tuple) else v.clone()
    return out


def _recording(ddpm, joint, log):
    """Wraps the graph getter: every replay logs the static state before and after it."""
    name, keys = ('_joint_graph', JOINT_KEYS) if joint else ('_graph', COND_KEYS)
    orig = getattr(ddpm, name)

    class Replay:
        def __init__(self, st, kind, g):
            self.st, self.kind, self.g = st, kind, g

        def replay(self):
            before = _snap(self.st, keys)
            self.g.replay()
            log.append(dict(kind=self.kind, st=self.st, before=before, after=_snap(self.st, keys)))

    def getter(st, kind, *a):
        return Replay(st, kind, orig(st, kind, *a))
    setattr(ddpm, name, getter)
    return lambda: delattr(ddpm, name)


def _check_draws(r, sampler, eta):
    """Draw ids of the round: (STAGE_LOOP, s, u, purpose) from the step counter and the round u."""
    s, u = int(r['before']['step']), int(r['before']['u'])
    want = [seeded.draw_id(seeded.STAGE_LOOP, s, u, p) for p in range(3)]
    assert r['after']['draw'].tolist() == want, (r['kind'], s, u)


def _check_cond_round(ddpm, r, sampler, eta, tables):
    st, b, a, kind = r['st'], r['before'], r['after'], r['kind']
    lm, pm, ip = st['lig_mask'], st['pocket_mask'], st['inpaint']
    s = int(b['step'])
    t_table, fast, anc = tables
    assert torch.equal(a['t'], t_table[s].expand_as(a['t']))
    with torch.no_grad():
        eps, _ = ddpm.dynamics(b['z'], b['pocket'], a['t'], lm, pm)
    renoise, commit = kind == 'inpaint_renoise', kind == 'inpaint_last'
    if sampler == 'ddim':
        cf, cr = a['coef_fast'], a['coef4']
        nrev = a['noise'] if eta > 0 else None
        if eta == 0:
            assert not a['noise'].any(), 'eta = 0 draws nothing'
        hist = torch.zeros_like(b['z'])
    else:
        cf, cr, nrev, hist = a['coef9'][:, :5], a['coef9'][:, 5:], None, b['hist']
    assert torch.equal(cf, fast[s].expand_as(cf)) and torch.equal(cr, anc[s, 3:].expand_as(cr))
    args = (b['z'], b['pocket'], hist, eps, nrev, a['noise1'], a['noise2'] if renoise else None, cf, cr, ip['known'], ip['com0'],
            ip['fixed'], lm, pm, sampler, commit)
    refs = [cond_round_ref(*args, d) for d in (torch.float32, torch.float64)]
    got = (a['z'], a['pocket']) + ((a['hist'],) if sampler == 'dpmpp_2m' else ())
    for i, x in enumerate(got):
        assert_fp64_bound(x, refs[0][i], refs[1][i], f'{sampler} eta={eta} {kind} s={s} u={int(b["u"])} output {i}')


def _inpaint_inputs(n_graphs=64, n_lig=25, n_fixed=10, seed=0):
    g = torch.Generator().manual_seed(1000 + seed)
    n = n_graphs * n_lig
    fixed = torch.zeros(n)
    fixed.view(n_graphs, n_lig)[:, :n_fixed] = 1
    lig = {'x': torch.randn((n, 3), generator=g) * 1.5,
           'one_hot': torch.nn.functional.one_hot(torch.randint(0, FULLATOM_COND.atom_nf, (n,), generator=g),
                                                  FULLATOM_COND.atom_nf).float(),
           'size': torch.full((n_graphs,), n_lig, dtype=torch.int64), 'mask': torch.repeat_interleave(torch.arange(n_graphs), n_lig)}
    return {k: v.cuda() for k, v in lig.items()}, fixed.cuda()


@pytest.fixture(scope='module')
def cond_model():
    ddpm = make_ddpm(FULLATOM_COND, False, timesteps=500)
    data = syn.synthetic_complex_batch(FULLATOM_COND, COND_LIG, COND_POC, seed=3)
    pocket = {'x': data['pocket_coords'].cuda(), 'one_hot': data['pocket_one_hot'].cuda(),
              'size': data['num_pocket_nodes'].cuda(), 'mask': data['pocket_mask'].cuda()}
    return ddpm, pocket


@pytest.mark.parametrize('resamplings', [1, 3])
@pytest.mark.parametrize('sampler,eta', RUNS)
def test_conditional_graph_rounds_teacher_forced(cond_model, sampler, eta, resamplings):
    ddpm, pocket = cond_model
    ligand, fixed = _inpaint_inputs()
    log = []
    undo = _recording(ddpm, False, log)
    try:
        out = ddpm.inpaint(ligand, {k: v.clone() for k, v in pocket.items()}, fixed, resamplings=resamplings, timesteps=N,
                           seeds=torch.arange(64) + 900, sampler=sampler, eta=eta)
    finally:
        undo()
    assert torch.isfinite(out[0]).all()
    assert len(log) == N * resamplings
    kinds = [r['kind'] for r in log]
    assert kinds == (['inpaint_renoise'] * (resamplings - 1) + ['inpaint_last']) * N
    assert [int(r['before']['step']) for r in log] == [s for s in range(N - 1, -1, -1) for _ in range(resamplings)]
    t_table, fast = ddpm._fast_tables(N, sampler, eta, 'cuda')
    _, anc = ddpm._schedule_tables(N, N, 'cuda')
    for r in log:
        _check_draws(r, sampler, eta)
        _check_cond_round(ddpm, r, sampler, eta, (t_table, fast, anc))


@pytest.fixture(scope='module')
def joint_model():
    ddpm = make_ddpm(FULLATOM_JOINT, True, timesteps=500)
    data = syn.synthetic_complex_batch(FULLATOM_JOINT, JOINT_LIG, JOINT_POC, seed=5)
    ligand = {'x': data['lig_coords'].cuda(), 'one_hot': data['lig_one_hot'].cuda(), 'size': data['num_lig_atoms'].cuda(),
              'mask': data['lig_mask'].cuda()}
    pocket = {'x': data['pocket_coords'].cuda(), 'one_hot': data['pocket_one_hot'].cuda(),
              'size': data['num_pocket_nodes'].cuda(), 'mask': data['pocket_mask'].cuda()}
    return ddpm, ligand, pocket


@pytest.mark.parametrize('sampler,eta,jump_length', [('ddim', 0.0, 1), ('ddim', 0.5, 1), ('dpmpp_2m', 0.0, 1),
                                                     ('ddim', 0.5, 2), ('ddim', 0.0, 2)])
def test_joint_graph_rounds_teacher_forced(joint_model, sampler, eta, jump_length):
    """The joint model generating for a fixed pocket (every pocket node fixed, no ligand atom fixed); with jump_length 1 the
    frames force the eager jump after an iteration that does not commit ('inpaint_hold' under 2M)."""
    ddpm, ligand, pocket = joint_model
    n = len(JOINT_LIG)
    log = []
    undo = _recording(ddpm, True, log)
    frames = 5 if jump_length == 1 else 1
    try:
        out = ddpm.inpaint({k: v.clone() for k, v in ligand.items()}, {k: v.clone() for k, v in pocket.items()},
                           torch.zeros(len(ligand['mask']), device='cuda'), torch.ones(len(pocket['mask']), device='cuda'),
                           resamplings=2, jump_length=jump_length, return_frames=frames, timesteps=N,
                           seeds=torch.arange(n) + 700, sampler=sampler, eta=eta)
    finally:
        undo()
    assert torch.isfinite(out[0]).all()
    kinds = {r['kind'] for r in log}
    assert kinds <= {'inpaint', 'inpaint_jump', 'inpaint_hold'} and 'inpaint_jump' in kinds
    assert ('inpaint_hold' in kinds) == (sampler == 'dpmpp_2m' and frames > 1)
    want, s = [], N - 1                         # the step of every iteration, as the eager loop walks the schedule
    schedule = ddpm.get_repaint_schedule(2, jump_length, N)
    for i, n_denoise in enumerate(schedule):
        for j in range(n_denoise):
            want.append(s)
            s += jump_length if (j == n_denoise - 1 and i < len(schedule) - 1) else 0
            s -= 1
    assert [int(r['before']['step']) for r in log] == want
    t_table, fast = ddpm._fast_tables(N, sampler, eta, 'cuda')
    _, anc = ddpm._joint_tables(N, jump_length, 'cuda')
    for r in log:
        st, b, a, kind = r['st'], r['before'], r['after'], r['kind']
        lm, pm, kn = st['lig_mask'], st['pocket_mask'], st['known']
        s = int(b['step'])
        _check_draws(r, sampler, eta)
        assert torch.equal(a['t'], t_table[s].expand_as(a['t']))
        with torch.no_grad():
            eps_l, eps_p = ddpm.dynamics(b['zl'], b['zp'], a['t'], lm, pm)
        jump, commit = kind == 'inpaint_jump', kind == 'inpaint'
        if sampler == 'ddim':
            cf, cr, nrev = a['coef_fast'], a['coef4'], (a['n_rev'] if eta > 0 else None)
            hl, hp = torch.zeros_like(b['zl']), torch.zeros_like(b['zp'])
        else:
            cf, cr, nrev = a['coef9'][:, :5], a['coef9'][:, 5:], None
            hl, hp = b['hist']
        assert torch.equal(cf, fast[s].expand_as(cf)) and torch.equal(cr, anc[s, 3:].expand_as(cr))
        args = (b['zl'], b['zp'], hl, hp, eps_l, eps_p, nrev, a['n_known'], a['n_jump'] if jump else None, cf, cr, kn['xl'],
                kn['xp'], kn['fl'], kn['fp'], lm, pm, sampler, commit)
        refs = [joint_round_ref(*args, d) for d in (torch.float32, torch.float64)]
        got = (a['zl'], a['zp']) + (a['hist'] if sampler == 'dpmpp_2m' else ())
        for i, x in enumerate(got):
            assert_fp64_bound(x, refs[0][i], refs[1][i], f'{sampler} eta={eta} j={jump_length} {kind} s={s} output {i}')


@pytest.mark.parametrize('denoising_steps', [10, 20])
@pytest.mark.parametrize('sampler,eta', [('ddim', 0.0), ('ddim', 0.5), ('dpmpp_2m', 0.0)])
def test_diversify_graph_steps_teacher_forced(cond_model, sampler, eta, denoising_steps):
    ddpm, pocket = cond_model
    ligand, _ = _inpaint_inputs()
    log = []
    undo = _recording(ddpm, False, log)
    try:
        out = ddpm.diversify(ligand, {k: v.clone() for k, v in pocket.items()}, 100, seeds=torch.arange(64) + 300,
                             sampler=sampler, eta=eta, denoising_steps=denoising_steps)
    finally:
        undo()
    assert torch.isfinite(out[0]).all() and len(log) == denoising_steps
    t_table, fast = ddpm._fast_tables(denoising_steps, sampler, eta, 'cuda', (100, ddpm.T))
    assert abs(float(t_table[-1]) - 100 / ddpm.T) < 1e-7
    for k, r in enumerate(log):
        st, b, a = r['st'], r['before'], r['after']
        lm, pm = st['lig_mask'], st['pocket_mask']
        s = int(b['step'])
        assert s == denoising_steps - 1 - k
        c = a['coef_fast']
        assert torch.equal(c, fast[s].expand_as(c)) and torch.equal(a['t'], t_table[s].expand_as(a['t']))
        with torch.no_grad():
            eps, _ = ddpm.dynamics(b['z'], b['pocket'], a['t'], lm, pm)
        if sampler == 'ddim':
            refs = [ddim_ref(b['z'], eps, a['noise'] if eta > 0 else None, c, b['pocket'], lm, pm, d)
                    for d in (torch.float32, torch.float64)]
            got = (a['z'], a['pocket'])
        else:
            refs = [multistep_ref(b['z'], eps, b['hist'], c, b['pocket'], lm, pm, d) for d in (torch.float32, torch.float64)]
            got = (a['z'], a['pocket'], a['hist'])
        for i, x in enumerate(got):
            assert_fp64_bound(x, refs[0][i], refs[1][i], f'diversify {sampler} K={denoising_steps} s={s} output {i}')


# ---- 3. regeneration ----------------------------------------------------------------------------------------------------
def _small(joint, engine):
    cfg = JOINT_CFG if joint else FULLATOM_COND.with_(n_layers=2)
    dyn = EGNNDynamics.from_config(cfg, device='cuda')
    dyn.load_state_dict(syn.synthetic_state_dict(cfg, 3))
    dyn.eval()
    dyn.math_mode = 'auto'
    dyn.deterministic = True
    cls = EnVariationalDiffusion if joint else ConditionalDDPM
    ddpm = cls(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=200,
               noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2', norm_values=(1, 4), size_histogram=HIST)
    ddpm.loop_engine = engine
    return ddpm.cuda().eval(), cfg


def _pick(d, idx):
    parts = [shard_pocket(d, i, i + 1) for i in idx]
    out = {k: torch.cat([p[k] for p in parts]) for k in ('x', 'one_hot', 'size')}
    out['mask'] = torch.cat([p['mask'] + j for j, p in enumerate(parts)])
    return out


def _runner(joint, engine, frames, **kw):
    ddpm, cfg = _small(joint, engine)
    g = torch.Generator().manual_seed(9)
    n_lig = torch.randint(2, 12, (64,), generator=g)
    n_poc = torch.randint(8, 40, (64,), generator=g)
    seeds = torch.arange(64) * 7919 + 3
    pocket = {k: v.cuda() for k, v in syn.synthetic_pocket(cfg, n_poc.tolist(), seed=4, spread=3.0).items()}
    lg = torch.Generator().manual_seed(10)
    n = int(n_lig.sum())
    ligand = {'x': torch.randn((n, 3), generator=lg).cuda() * 1.5,
              'one_hot': torch.nn.functional.one_hot(torch.randint(0, cfg.atom_nf, (n,), generator=lg), cfg.atom_nf).float().cuda(),
              'size': n_lig.cuda(), 'mask': torch.repeat_interleave(torch.arange(64), n_lig).cuda()}
    fixed = torch.cat([(torch.arange(k) < 2).float() for k in n_lig.tolist()]).cuda()

    def run(idx, **k2):
        lig, poc = _pick(ligand, idx), _pick(pocket, idx)
        f = torch.cat([fixed[ligand['mask'] == i] for i in idx])
        args = {**kw, **k2}
        if joint:
            return ddpm.inpaint(lig, poc, torch.zeros_like(f), torch.ones(len(poc['mask']), device='cuda'), resamplings=2,
                                return_frames=frames, seeds=seeds[idx], **args)
        return ddpm.inpaint(lig, poc, f, resamplings=2, return_frames=frames, seeds=seeds[idx], **args)
    return ddpm, run


def _rows(out, mask, g, frames):
    return out[:, mask == g] if frames > 1 else out[mask == g]


@pytest.mark.parametrize('engine', ['graph', 'eager'])
@pytest.mark.parametrize('sampler,eta', [('ddim', 0.0), ('ddim', 0.5), ('dpmpp_2m', 0.0)])
@pytest.mark.parametrize('joint', [False, True], ids=['cond', 'joint'])
def test_regenerate_graphs_alone_and_reversed(joint, sampler, eta, engine):
    frames = 5
    _, run = _runner(joint, engine, frames, sampler=sampler, eta=eta, timesteps=10)
    full = run(list(range(64)))
    assert torch.isfinite(full[0]).all()
    for idx in ([0], [37], [63], [63, 37, 0]):
        sub = run(idx)
        for k, g in enumerate(idx):
            for part, mi in ((0, 2), (1, 3)):
                assert torch.equal(_rows(sub[part], sub[mi], k, frames), _rows(full[part], full[mi], g, frames)), \
                    (sampler, eta, engine, idx, g, part)


# ---- 4. re-capture, tables, the default, NaN ----------------------------------------------------------------------------
@pytest.mark.parametrize('joint', [False, True], ids=['cond', 'joint'])
def test_sampler_switch_recaptures_and_default_is_ddpm(joint):
    ddpm, run = _runner(joint, 'graph', 1, timesteps=10)
    cache = lambda: ddpm._joint_cache if joint else ddpm._graph_cache
    idx = list(range(64))
    a = run(idx, sampler='ddim', eta=0.5)
    st_a = next(iter(cache().values()))
    b = run(idx, sampler='dpmpp_2m')
    st_b = next(iter(cache().values()))
    assert st_b is not st_a and len(cache()) == 1
    c = run(idx, sampler='ddim', eta=0.5)
    assert next(iter(cache().values())) is not st_b
    assert all(torch.equal(x, y) for x, y in zip(a, c)), 'switching back to ddim changed the bits'
    assert not torch.equal(a[0], b[0])
    d, e = run(idx), run(idx, sampler='ddpm')
    assert all(torch.equal(x, y) for x, y in zip(d, e)), "sampler='ddpm' differs from the default call"


def test_diversify_tables_follow_noising_steps(cond_model):
    ddpm, pocket = cond_model
    ligand, _ = _inpaint_inputs()
    seeds = torch.arange(64) + 40
    call = lambda n, **kw: ddpm.diversify({k: v.clone() for k, v in ligand.items()}, {k: v.clone() for k, v in pocket.items()},
                                          n, seeds=seeds, **kw)
    a = call(100, sampler='dpmpp_2m', denoising_steps=10)
    st = next(iter(ddpm._graph_cache.values()))
    want_t, want = ddpm._fast_tables(10, 'dpmpp_2m', 0.0, 'cuda', (100, ddpm.T))
    assert torch.equal(st['fast_t'], want_t) and torch.equal(st['fast_table'], want)
    b = call(200, sampler='dpmpp_2m', denoising_steps=10)
    st2 = next(iter(ddpm._graph_cache.values()))
    want_t, want = ddpm._fast_tables(10, 'dpmpp_2m', 0.0, 'cuda', (200, ddpm.T))
    assert st2 is not st and torch.equal(st2['fast_t'], want_t) and torch.equal(st2['fast_table'], want)
    assert not torch.equal(a[0], b[0])
    assert all(torch.equal(x, y) for x, y in zip(a, call(100, sampler='dpmpp_2m', denoising_steps=10)))
    assert all(torch.equal(x, y) for x, y in zip(call(20), call(20, sampler='ddpm', denoising_steps=20)))


@pytest.mark.parametrize('engine', ['graph', 'eager'])
@pytest.mark.parametrize('sampler', ['ddpm', 'ddim', 'dpmpp_2m'])
def test_nan_reports_as_for_the_ancestral_sampler(sampler, engine):
    ddpm, cfg = _small(False, engine)
    pocket = {k: v.cuda() for k, v in syn.synthetic_pocket(cfg, [20, 14], seed=2, spread=3.0).items()}
    ligand = {'x': torch.randn(9, 3).cuda(), 'one_hot': torch.nn.functional.one_hot(torch.arange(9) % cfg.atom_nf,
                                                                                    cfg.atom_nf).float().cuda(),
              'size': torch.tensor([5, 4]).cuda(), 'mask': torch.tensor([0] * 5 + [1] * 4).cuda()}
    fixed = torch.tensor([1., 1., 0., 0., 0., 1., 0., 0., 0.]).cuda()
    bad = {k: v.clone() for k, v in pocket.items()}
    bad['one_hot'] = bad['one_hot'].float()
    bad['one_hot'][3, 1] = float('nan')
    with pytest.raises(ValueError, match='NaN detected in EGNN output'):
        ddpm.inpaint({k: v.clone() for k, v in ligand.items()}, bad, fixed, resamplings=2, timesteps=6, sampler=sampler)
    out = ddpm.inpaint({k: v.clone() for k, v in ligand.items()}, pocket, fixed, resamplings=2, timesteps=6, sampler=sampler)
    assert torch.isfinite(out[0]).all()
