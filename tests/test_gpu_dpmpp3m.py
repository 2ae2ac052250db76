"""GPU: the third-order multistep sampler 'dpmpp_3m' (DESIGN §15).

1. dsb_ddpm_multistep3_update and dsb_ddpm_multistep3_inpaint_update, both model variants, against float64 on every output
   (z, pocket, both histories): configs[2] and a ragged batch with an empty pocket and a one-atom ligand; a first step
   (neither history read), a second step (m2 not read) and a later step; commit 0 and 1, re-noise on and off.  Repeats bit for
   bit, and a graph's result does not depend on its batch.
2. The graph engine, teacher-forced replay by replay against float64 along seeded 50- and 20-step runs: sampling on
   configs[2] (3xFP16) and on the joint production model, conditional inpainting (3 resamplings), the joint model generating
   for a fixed pocket (2 resamplings, frames forcing the eager jump) and diversify.  Every replay's denoiser output is
   recomputed on the recorded state (deterministic mode: the same bits).  Frames land at the ancestral sampler's steps.
3. Seeded deterministic runs, both engines, both models: graphs 0, 37, 63 alone and in a reversed sub-batch equal the full
   batch in every frame, and a repeated run repeats the bits; 2M -> 3M -> 2M re-captures and replays the first 2M run's bits.
4. A NaN reports as it does for the ancestral sampler.
"""
import ctypes as C

import pytest
import torch

from ddpm_cases import HIST, JOINT_CFG, assert_fp64_bound
from dpmpp3m_cases import cond_round3_ref, joint_multistep3_ref, joint_round3_ref, multistep3_ref
from trajectory_cases import COND_LIG, COND_POC, JOINT_LIG, JOINT_POC, full_pocket, make_ddpm
from diffsbdd_b200 import _native, synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM
from diffsbdd_b200.config import FULLATOM_COND, FULLATOM_JOINT
from diffsbdd_b200.distributed import shard_pocket
from diffsbdd_b200.dynamics import EGNNDynamics
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion

pytestmark = pytest.mark.gpu
N = 50
SHAPES = {'configs2': ([25] * 64, [175] * 64), 'ragged': ([7, 1, 12, 3, 9], [30, 0, 9, 140, 11])}
STEPS = {'first': N - 1, 'second': N - 2, 'later': 20}


# ---- 1. the kernels -----------------------------------------------------------------------------------------------------
def _buffers(joint, shape, seed):
    cfg = FULLATOM_JOINT if joint else FULLATOM_COND
    A, R = cfg.atom_nf, cfg.residue_nf
    n_lig, n_poc = SHAPES[shape]
    n, dev = len(n_lig), 'cuda'
    g = torch.Generator(device=dev).manual_seed(seed)
    lm = torch.repeat_interleave(torch.arange(n, device=dev), torch.tensor(n_lig, device=dev))
    pm = torch.repeat_interleave(torch.arange(n, device=dev), torch.tensor(n_poc, device=dev))
    rnd = lambda r, c, s=1.0: torch.randn((r, c), device=dev, generator=g) * s
    NL, NP = len(lm), len(pm)
    fl = (torch.rand(NL, device=dev, generator=g) < 0.4).float()
    fp = (torch.rand(NP, device=dev, generator=g) < 0.7).float()
    if shape == 'ragged':                       # graph 2: every node fixed; graph 4: none
        fl[lm == 2], fp[pm == 2], fl[lm == 4], fp[pm == 4] = 1., 1., 0., 0.
    b = dict(zl=rnd(NL, 3 + A), zp=rnd(NP, 3 + R, 4.0), h1l=rnd(NL, 3 + A, 2.0), h1p=rnd(NP, 3 + R, 2.0),
             h2l=rnd(NL, 3 + A, 2.0), h2p=rnd(NP, 3 + R, 2.0), el=rnd(NL, 3 + A), ep=rnd(NP, 3 + R), xl=rnd(NL, 3 + A, 1.5),
             xp=rnd(NP, 3 + R, 3.0), com0=rnd(n, 3), fl=fl, fp=fp, nk=(rnd(NL + NP, 3), rnd(NL, A), rnd(NP, R)),
             nr=(rnd(NL + NP, 3), rnd(NL, A), rnd(NP, R)), nkc=rnd(NL, 3 + A), nrc=rnd(NL, 3 + A))
    return b, lm, pm, A, R


def _rows(step, n, with_repaint):
    ddpm = make_ddpm(FULLATOM_COND.with_(n_layers=1), False, timesteps=500)
    _, table = ddpm._fast_tables(N, 'dpmpp_3m', 0.0, 'cuda')
    if with_repaint:
        _, anc = ddpm._schedule_tables(N, N, 'cuda')
        table = torch.cat((table, anc[:, 3:]), 1)
    # every graph takes the row of `step` except graphs 1 and 3, which take later rows: rows differ per graph
    rows = torch.tensor([STEPS[step], 30, STEPS[step], 5, STEPS[step]], device='cuda')
    return table[rows[torch.arange(n, device='cuda') % 5]].contiguous()


def _step_kernel(joint, b, coef, lm, pm, A, R):
    """dsb_ddpm_multistep3_update on copies; returns (z_lig, z_pocket, m1_lig, m1_pocket, m2_lig, m2_pocket) (conditional:
    the pocket histories are None)."""
    zl, zp, h1l, h2l = (b[k].clone() for k in ('zl', 'zp', 'h1l', 'h2l'))
    h1p, h2p = (b['h1p'].clone(), b['h2p'].clone()) if joint else (None, None)
    P = lambda x: None if x is None else x.data_ptr()
    _native.check(_native.load().dsb_ddpm_multistep3_update(
        P(zl), P(zp), P(h1l), P(h1p), P(h2l), P(h2p), P(b['el']), P(b['ep']) if joint else None, P(coef), P(lm), P(pm),
        zl.shape[0], zp.shape[0], coef.shape[0], A, R, int(joint), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return zl, zp, h1l, h1p, h2l, h2p


def _round_kernel(joint, b, coef, lm, pm, A, R, renoise, commit):
    """dsb_ddpm_multistep3_inpaint_update on copies; outputs as _step_kernel."""
    zl, zp, h1l, h2l = (b[k].clone() for k in ('zl', 'zp', 'h1l', 'h2l'))
    h1p, h2p = (b['h1p'].clone(), b['h2p'].clone()) if joint else (None, None)
    P = lambda x: None if x is None else x.data_ptr()
    if joint:
        n3 = b['nr'] if renoise else (None, None, None)
        args = (P(b['el']), P(b['ep']), P(b['xl']), P(b['xp']), None, P(b['fl']), P(b['fp']), *[P(x) for x in b['nk']],
                *[P(x) for x in n3])
    else:
        args = (P(b['el']), None, P(b['xl']), None, P(b['com0']), P(b['fl']), None, P(b['nkc']), None, None,
                P(b['nrc']) if renoise else None, None, None)
    _native.check(_native.load().dsb_ddpm_multistep3_inpaint_update(
        P(zl), P(zp), P(h1l), P(h1p), P(h2l), P(h2p), *args, P(coef), P(lm), P(pm), zl.shape[0], zp.shape[0], coef.shape[0],
        A, R, int(joint), int(commit), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return zl, zp, h1l, h1p, h2l, h2p


NAMES = ('z_lig', 'z_pocket', 'm1_lig', 'm1_pocket', 'm2_lig', 'm2_pocket')


def _compare(got, refs, what, nan_rows=None):
    """Every output within the float64 bound; ``nan_rows[k]``: rows of output k that must still hold the NaN they came in
    with (a history that was neither read nor replaced), left out of the comparison."""
    for k, name in enumerate(NAMES):
        if got[k] is None:
            continue
        x, r32, r64 = got[k], refs[0][k], refs[1][k]
        if nan_rows is not None and nan_rows[k] is not None:
            m = nan_rows[k]
            assert torch.isnan(x[m]).all(), f'{what} {name}: an unread history changed'
            x, r32, r64 = x[~m], r32[~m], r64[~m]
        assert torch.isfinite(x).all(), f'{what} {name}'
        assert_fp64_bound(x, r32, r64, f'{what} {name}')


def _unread(b, step, lm, pm):
    """The inputs with the histories a step must not read set to NaN in the graphs that take the step's row (g % 5 in 0, 2,
    4), the same inputs with them zeroed (the reference), and per history key the NaN rows."""
    nan, zero, rows = dict(b), dict(b), {}
    keys = ('h1l', 'h1p', 'h2l', 'h2p') if step == 'first' else ('h2l', 'h2p') if step == 'second' else ()
    for k in keys:
        m = (lm if k.endswith('l') else pm) % 5
        m = (m == 0) | (m == 2) | (m == 4)
        nan[k], zero[k] = b[k].clone(), b[k].clone()
        nan[k][m], zero[k][m] = float('nan'), 0.0
        rows[k] = m
    return nan, zero, rows


def _graph1(b, lm, pm):
    NL, NP = len(lm), len(pm)
    l1, p1 = lm == 1, pm == 1
    pick = lambda x: x[torch.cat((l1, p1))] if x.shape[0] == NL + NP else x[l1] if x.shape[0] == NL else x[p1]
    return {k: (tuple(pick(x) for x in v) if isinstance(v, tuple) else v[1:2] if k == 'com0' else pick(v))
            for k, v in b.items()}, lm[l1] - 1, pm[p1] - 1, l1, p1


@pytest.mark.parametrize('step', list(STEPS))
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('joint', [False, True], ids=['cond', 'joint'])
def test_multistep3_kernel_against_float64(joint, shape, step):
    b, lm, pm, A, R = _buffers(joint, shape, 7)
    coef = _rows(step, len(SHAPES[shape][0]), False)
    nan, zero, _ = _unread(b, step, lm, pm)
    got = _step_kernel(joint, nan, coef, lm, pm, A, R)
    if joint:
        refs = [joint_multistep3_ref(zero['zl'], zero['zp'], zero['el'], zero['ep'], zero['h1l'], zero['h1p'], zero['h2l'],
                                     zero['h2p'], coef, lm, pm, d) for d in (torch.float32, torch.float64)]
    else:
        refs = [multistep3_ref(zero['zl'], zero['el'], zero['h1l'], zero['h2l'], coef, zero['zp'], lm, pm, d)
                for d in (torch.float32, torch.float64)]
        refs = [(r[0], r[1], r[2], None, r[3], None) for r in refs]
        assert torch.equal(got[1][:, 3:], b['zp'][:, 3:]), 'the conditional pocket features must not change'
    _compare(got, refs, f'{shape} {step}')
    again = _step_kernel(joint, nan, coef, lm, pm, A, R)
    assert all(x is None or torch.equal(x, y) for x, y in zip(got, again))
    sub, lm1, pm1, l1, p1 = _graph1(nan, lm, pm)
    one = _step_kernel(joint, sub, coef[1:2].contiguous(), lm1, pm1, A, R)
    for k, rows in enumerate((l1, p1, l1, p1, l1, p1)):
        if got[k] is not None:
            assert torch.equal(one[k], got[k][rows]), f'{shape} {step}: graph 1 alone, {NAMES[k]}'


@pytest.mark.parametrize('step', list(STEPS))
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('joint', [False, True], ids=['cond', 'joint'])
def test_multistep3_inpaint_kernel_against_float64(joint, shape, step):
    b, lm, pm, A, R = _buffers(joint, shape, 8)
    coef = _rows(step, len(SHAPES[shape][0]), True)
    nan, zero, unread = _unread(b, step, lm, pm)
    cf, cr = coef[:, :6], coef[:, 6:]
    for renoise, commit in ((True, False), (False, True), (True, True), (False, False)):
        got = _round_kernel(joint, nan, coef, lm, pm, A, R, renoise, commit)
        what = f'{shape} {step} renoise={renoise} commit={commit}'
        z = zero
        if joint:
            args = (z['zl'], z['zp'], z['h1l'], z['h1p'], z['h2l'], z['h2p'], z['el'], z['ep'], z['nk'],
                    z['nr'] if renoise else None, cf, cr, z['xl'], z['xp'], z['fl'], z['fp'], lm, pm, commit)
            refs = [joint_round3_ref(*args, d) for d in (torch.float32, torch.float64)]
        else:
            args = (z['zl'], z['zp'], z['h1l'], z['h2l'], z['el'], z['nkc'], z['nrc'] if renoise else None, cf, cr, z['xl'],
                    z['com0'], z['fl'], lm, pm, commit)
            refs = [(r[0], r[1], r[2], None, r[3], None) for r in (cond_round3_ref(*args, d) for d in (torch.float32, torch.float64))]
            assert torch.equal(got[1][:, 3:], b['zp'][:, 3:]), 'the conditional pocket features must not change'
        # a round that does not commit keeps an unread NaN history NaN (translated); one that commits replaces it
        nan_rows = [None if commit else unread.get(key) for key in ('zl', 'zp', 'h1l', 'h1p', 'h2l', 'h2p')]
        _compare(got, refs, what, nan_rows)
        if not commit:
            for k, key in ((2, 'h1l'), (4, 'h2l')):
                assert torch.equal(got[k][:, 3:].nan_to_num(), nan[key][:, 3:].nan_to_num()), \
                    f'{what}: a round that does not commit only translates'
        again = _round_kernel(joint, nan, coef, lm, pm, A, R, renoise, commit)
        assert all(x is None or torch.equal(x.nan_to_num(), y.nan_to_num()) for x, y in zip(got, again))
        sub, lm1, pm1, l1, p1 = _graph1(nan, lm, pm)
        one = _round_kernel(joint, sub, coef[1:2].contiguous(), lm1, pm1, A, R, renoise, commit)
        for k, rows in enumerate((l1, p1, l1, p1, l1, p1)):
            if got[k] is not None:
                assert torch.equal(one[k], got[k][rows]), f'{what}: graph 1 alone, {NAMES[k]}'


# ---- 2. the graph engine, teacher-forced --------------------------------------------------------------------------------
COND_KEYS = ('z', 'pocket', 'hist', 'hist2', 'noise1', 'noise2', 't', 'coef_fast', 'coef10', 'step')
JOINT_KEYS = ('zl', 'zp', 'hist', 'hist2', 'n_known', 'n_jump', 't', 'coef_fast', 'coef10', 'step')


def _snap(st, keys):
    return {k: (tuple(x.clone() for x in st[k]) if isinstance(st[k], tuple) else st[k].clone()) for k in keys if k in st}


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

    setattr(ddpm, name, lambda st, kind, *a: Replay(st, kind, orig(st, kind, *a)))
    return lambda: delattr(ddpm, name)


def _check_step(ddpm, joint, r, table, t_table):
    """A plain 3M replay (sampling, diversify) against float64."""
    st, b, a = r['st'], r['before'], r['after']
    lm, pm, s = st['lig_mask'], st['pocket_mask'], int(b['step'])
    c = a['coef_fast']
    assert torch.equal(c, table[s].expand_as(c)) and torch.equal(a['t'], t_table[s].expand_as(a['t']))
    with torch.no_grad():
        if joint:
            eps_l, eps_p = ddpm.dynamics(b['zl'], b['zp'], a['t'], lm, pm)
            (h1l, h1p), (h2l, h2p) = b['hist'], b['hist2']
            refs = [joint_multistep3_ref(b['zl'], b['zp'], eps_l, eps_p, h1l, h1p, h2l, h2p, c, lm, pm, d)
                    for d in (torch.float32, torch.float64)]
            got = (a['zl'], a['zp'], a['hist'][0], a['hist'][1], a['hist2'][0], a['hist2'][1])
        else:
            eps, _ = ddpm.dynamics(b['z'], b['pocket'], a['t'], lm, pm)
            refs = [multistep3_ref(b['z'], eps, b['hist'], b['hist2'], c, b['pocket'], lm, pm, d)
                    for d in (torch.float32, torch.float64)]
            got = (a['z'], a['pocket'], a['hist'], a['hist2'])
    for i, x in enumerate(got):
        assert_fp64_bound(x, refs[0][i], refs[1][i], f'3M s={s} output {i}')


@pytest.fixture(scope='module', params=['cond', 'joint'])
def model(request):
    joint = request.param == 'joint'
    ddpm = make_ddpm(FULLATOM_JOINT if joint else FULLATOM_COND, joint, timesteps=500)
    inputs = (torch.tensor(JOINT_LIG).cuda(), torch.tensor(JOINT_POC).cuda()) if joint else full_pocket()
    return joint, ddpm, inputs, torch.arange(500, 500 + len(inputs[1]))


@pytest.mark.parametrize('steps', [50, 20])
def test_sampling_teacher_forced(model, steps):
    joint, ddpm, inputs, seeds = model
    frames, log = 5, []
    undo = _recording(ddpm, joint, log)
    try:
        if joint:
            out = ddpm.sample(len(inputs[0]), *inputs, return_frames=frames, timesteps=steps, device='cuda', seeds=seeds,
                              sampler='dpmpp_3m')
        else:
            out = ddpm.sample_given_pocket({k: v.clone() for k, v in inputs[0].items()}, inputs[1], return_frames=frames,
                                           timesteps=steps, seeds=seeds, sampler='dpmpp_3m')
    finally:
        undo()
    assert torch.isfinite(out[0]).all()
    assert [int(r['before']['step']) for r in log] == list(range(steps - 1, -1, -1))
    t_table, table = ddpm._fast_tables(steps, 'dpmpp_3m', 0.0, 'cuda')
    zk, pk = ('zl', 'zp') if joint else ('z', 'pocket')
    for r in log:
        _check_step(ddpm, joint, r, table, t_table)
        s = int(r['before']['step'])
        if s % (steps // frames) == 0 and s > 0:     # frames at the ancestral sampler's steps (frame 0 is the final sample)
            lig, poc = ddpm.unnormalize_z(r['after'][zk], r['after'][pk])
            assert torch.equal(out[0][s // (steps // frames)], lig) and torch.equal(out[1][s // (steps // frames)], poc)


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


@pytest.mark.parametrize('steps', [50, 20])
def test_conditional_inpaint_teacher_forced(cond_model, steps):
    ddpm, pocket = cond_model
    ligand, fixed = _inpaint_inputs()
    resamplings, log = 3, []
    undo = _recording(ddpm, False, log)
    try:
        out = ddpm.inpaint(ligand, {k: v.clone() for k, v in pocket.items()}, fixed, resamplings=resamplings, timesteps=steps,
                           seeds=torch.arange(64) + 900, sampler='dpmpp_3m')
    finally:
        undo()
    assert torch.isfinite(out[0]).all()
    assert [r['kind'] for r in log] == (['inpaint_renoise'] * (resamplings - 1) + ['inpaint_last']) * steps
    assert [int(r['before']['step']) for r in log] == [s for s in range(steps - 1, -1, -1) for _ in range(resamplings)]
    t_table, fast = ddpm._fast_tables(steps, 'dpmpp_3m', 0.0, 'cuda')
    _, anc = ddpm._schedule_tables(steps, steps, 'cuda')
    for r in log:
        st, b, a, kind = r['st'], r['before'], r['after'], r['kind']
        lm, pm, ip, s = st['lig_mask'], st['pocket_mask'], st['inpaint'], int(b['step'])
        assert torch.equal(a['t'], t_table[s].expand_as(a['t']))
        cf, cr = a['coef10'][:, :6], a['coef10'][:, 6:]
        assert torch.equal(cf, fast[s].expand_as(cf)) and torch.equal(cr, anc[s, 3:].expand_as(cr))
        with torch.no_grad():
            eps, _ = ddpm.dynamics(b['z'], b['pocket'], a['t'], lm, pm)
        renoise = kind == 'inpaint_renoise'
        args = (b['z'], b['pocket'], b['hist'], b['hist2'], eps, a['noise1'], a['noise2'] if renoise else None, cf, cr,
                ip['known'], ip['com0'], ip['fixed'], lm, pm, not renoise)
        refs = [cond_round3_ref(*args, d) for d in (torch.float32, torch.float64)]
        for i, x in enumerate((a['z'], a['pocket'], a['hist'], a['hist2'])):
            assert_fp64_bound(x, refs[0][i], refs[1][i], f'3M {kind} s={s} output {i}')


@pytest.fixture(scope='module')
def joint_model():
    ddpm = make_ddpm(FULLATOM_JOINT, True, timesteps=500)
    data = syn.synthetic_complex_batch(FULLATOM_JOINT, JOINT_LIG, JOINT_POC, seed=5)
    ligand = {'x': data['lig_coords'].cuda(), 'one_hot': data['lig_one_hot'].cuda(), 'size': data['num_lig_atoms'].cuda(),
              'mask': data['lig_mask'].cuda()}
    pocket = {'x': data['pocket_coords'].cuda(), 'one_hot': data['pocket_one_hot'].cuda(),
              'size': data['num_pocket_nodes'].cuda(), 'mask': data['pocket_mask'].cuda()}
    return ddpm, ligand, pocket


@pytest.mark.parametrize('steps', [50, 20])
def test_joint_inpaint_teacher_forced(joint_model, steps):
    """The joint model generating for a fixed pocket; the frames force the eager jump after an 'inpaint_hold' iteration."""
    ddpm, ligand, pocket = joint_model
    log = []
    undo = _recording(ddpm, True, log)
    try:
        out = ddpm.inpaint({k: v.clone() for k, v in ligand.items()}, {k: v.clone() for k, v in pocket.items()},
                           torch.zeros(len(ligand['mask']), device='cuda'), torch.ones(len(pocket['mask']), device='cuda'),
                           resamplings=2, jump_length=1, return_frames=5, timesteps=steps,
                           seeds=torch.arange(len(JOINT_LIG)) + 700, sampler='dpmpp_3m')
    finally:
        undo()
    assert torch.isfinite(out[0]).all()
    kinds = {r['kind'] for r in log}
    assert kinds == {'inpaint', 'inpaint_jump', 'inpaint_hold'}
    t_table, fast = ddpm._fast_tables(steps, 'dpmpp_3m', 0.0, 'cuda')
    _, anc = ddpm._joint_tables(steps, 1, 'cuda')
    for r in log:
        st, b, a, kind = r['st'], r['before'], r['after'], r['kind']
        lm, pm, kn, s = st['lig_mask'], st['pocket_mask'], st['known'], int(b['step'])
        assert torch.equal(a['t'], t_table[s].expand_as(a['t']))
        cf, cr = a['coef10'][:, :6], a['coef10'][:, 6:]
        assert torch.equal(cf, fast[s].expand_as(cf)) and torch.equal(cr, anc[s, 3:].expand_as(cr))
        with torch.no_grad():
            eps_l, eps_p = ddpm.dynamics(b['zl'], b['zp'], a['t'], lm, pm)
        jump = kind == 'inpaint_jump'
        args = (b['zl'], b['zp'], *b['hist'], *b['hist2'], eps_l, eps_p, a['n_known'], a['n_jump'] if jump else None, cf, cr,
                kn['xl'], kn['xp'], kn['fl'], kn['fp'], lm, pm, kind == 'inpaint')
        refs = [joint_round3_ref(*args, d) for d in (torch.float32, torch.float64)]
        got = (a['zl'], a['zp'], *a['hist'], *a['hist2'])
        for i, x in enumerate(got):
            assert_fp64_bound(x, refs[0][i], refs[1][i], f'3M {kind} s={s} output {i}')


@pytest.mark.parametrize('steps', [10, 20])
def test_diversify_teacher_forced(cond_model, steps):
    ddpm, pocket = cond_model
    ligand, _ = _inpaint_inputs()
    log = []
    undo = _recording(ddpm, False, log)
    try:
        out = ddpm.diversify(ligand, {k: v.clone() for k, v in pocket.items()}, 100, seeds=torch.arange(64) + 300,
                             sampler='dpmpp_3m', denoising_steps=steps)
    finally:
        undo()
    assert torch.isfinite(out[0]).all() and [int(r['before']['step']) for r in log] == list(range(steps - 1, -1, -1))
    t_table, fast = ddpm._fast_tables(steps, 'dpmpp_3m', 0.0, 'cuda', (100, ddpm.T))
    for r in log:
        _check_step(ddpm, False, r, fast, t_table)


# ---- 3. regeneration, determinism, re-capture ---------------------------------------------------------------------------
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
    n_lig = torch.randint(1, 12, (64,), generator=g).cuda()
    n_poc = torch.randint(8, 40, (64,), generator=g).cuda()
    seeds = torch.arange(64) * 7919 + 3
    if joint:
        run = lambda idx, **k2: ddpm.sample(len(idx), n_lig[idx], n_poc[idx], return_frames=frames, device='cuda',
                                            seeds=seeds[idx], **{**kw, **k2})
    else:
        pocket = {k: v.cuda() for k, v in syn.synthetic_pocket(cfg, n_poc.tolist(), seed=4, spread=3.0).items()}
        run = lambda idx, **k2: ddpm.sample_given_pocket(_pick({k: v.clone() for k, v in pocket.items()}, idx), n_lig[idx],
                                                         return_frames=frames, seeds=seeds[idx], **{**kw, **k2})
    return ddpm, run


def _graph_rows(out, mask, g, frames):
    return out[:, mask == g] if frames > 1 else out[mask == g]


@pytest.mark.parametrize('engine', ['graph', 'eager'])
@pytest.mark.parametrize('joint', [False, True], ids=['cond', 'joint'])
def test_regenerate_graphs_alone_and_reversed(joint, engine):
    frames = 5
    _, run = _runner(joint, engine, frames, sampler='dpmpp_3m', timesteps=N)
    full = run(list(range(64)))
    assert torch.isfinite(full[0]).all()
    again = run(list(range(64)))
    assert all(torch.equal(a, b) for a, b in zip(full, again)), 'a deterministic seeded run did not repeat bit for bit'
    for idx in ([0], [37], [63], [63, 37, 0]):
        sub = run(idx)
        for k, g in enumerate(idx):
            for part, mi in ((0, 2), (1, 3)):
                assert torch.equal(_graph_rows(sub[part], sub[mi], k, frames), _graph_rows(full[part], full[mi], g, frames)), \
                    (engine, idx, g, part)


@pytest.mark.parametrize('joint', [False, True], ids=['cond', 'joint'])
def test_2m_3m_2m_recaptures_and_replays_the_same_bits(joint):
    ddpm, run = _runner(joint, 'graph', 1, timesteps=N)
    cache = lambda: ddpm._joint_cache if joint else ddpm._graph_cache
    idx = list(range(64))
    a = run(idx, sampler='dpmpp_2m')
    st_a = next(iter(cache().values()))
    b = run(idx, sampler='dpmpp_3m')
    st_b = next(iter(cache().values()))
    assert st_b is not st_a and 'dpmpp_3m' in st_b['graphs'] and len(cache()) == 1
    c = run(idx, sampler='dpmpp_2m')
    assert next(iter(cache().values())) is not st_b
    assert all(torch.equal(x, y) for x, y in zip(a, c)), 'switching back to dpmpp_2m changed the bits'
    assert not torch.equal(a[0], b[0])


# ---- 4. NaN status ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('engine', ['graph', 'eager'])
def test_nan_reports_as_for_the_ancestral_sampler(engine):
    ddpm, cfg = _small(False, engine)
    pocket = {k: v.cuda() for k, v in syn.synthetic_pocket(cfg, [20, 14], seed=2, spread=3.0).items()}
    bad = {k: v.clone() for k, v in pocket.items()}
    bad['one_hot'] = bad['one_hot'].float()
    bad['one_hot'][3, 1] = float('nan')
    n_lig = torch.tensor([5, 4]).cuda()
    with pytest.raises(ValueError, match='NaN detected in EGNN output'):
        ddpm.sample_given_pocket(bad, n_lig, timesteps=10, sampler='dpmpp_3m')
    out = ddpm.sample_given_pocket(pocket, n_lig, timesteps=10, sampler='dpmpp_3m')     # the sticky flag was cleared
    assert torch.isfinite(out[0]).all()
