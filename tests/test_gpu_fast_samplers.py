"""GPU: the few-step samplers 'ddim' and 'dpmpp_2m' (DESIGN §13).

1. dsb_ddpm_multistep_update, both variants, against float64 on every output (z, pocket, history): configs[2], a ragged
   batch with an empty pocket and a one-atom ligand; a first step (w = 0, history not read) and a later step.
2. The graph engine, teacher-forced step by step against float64 along seeded 50-step trajectories (DDIM at eta 0 and 0.5,
   2M) on configs[2] (3xFP16) and the joint production model; the captured step is recorded as tests/trajectory_cases.py
   does, and the denoiser output is recomputed on the recorded state (deterministic mode: the same bits).  Frames land at
   the steps the ancestral sampler saves them at.
3. With seeds, each teacher-forced DDIM eta = 1 step draws the ancestral step's noise and both are within the fp32 bound of
   the same float64 step.
4. Seeded deterministic runs of every new sampler, both engines, both models: graphs 0, 37, 63 alone and in a reversed
   sub-batch equal the full batch in every frame; a sampler switch re-captures and switching back repeats the bits;
   sampler='ddpm' equals the default call.
5. A NaN reports as it does for the ancestral sampler.
"""
import ctypes as C

import pytest
import torch

from ddpm_cases import HIST, JOINT_CFG, assert_fp64_bound
from fast_sampler_cases import ddim_ref, joint_ddim_ref, joint_multistep_ref, multistep_ref
from trajectory_cases import JOINT_LIG, JOINT_POC, full_pocket, joint_update, ligand_update, make_ddpm
from diffsbdd_b200 import _native, seeded, synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM
from diffsbdd_b200.config import FULLATOM_COND, FULLATOM_JOINT
from diffsbdd_b200.distributed import shard_pocket
from diffsbdd_b200.dynamics import EGNNDynamics
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion

pytestmark = pytest.mark.gpu
N = 50
RUNS = [('ddim', 0.0), ('ddim', 0.5), ('dpmpp_2m', 0.0)]


# ---- 1. the kernel ------------------------------------------------------------------------------------------------------
def multistep(zl, zp, hl, hp, eps_l, eps_p, coef, lm, pm, A, R, joint):
    """dsb_ddpm_multistep_update on copies; returns (z_lig, z_pocket, hist_lig[, hist_pocket])."""
    zl, zp, hl = zl.clone(), zp.clone(), hl.clone()
    hp = hp.clone() if joint else None
    P = lambda x: None if x is None else x.data_ptr()
    _native.check(_native.load().dsb_ddpm_multistep_update(
        P(zl), P(zp), P(hl), P(hp), P(eps_l), P(eps_p) if joint else None, P(coef), P(lm), P(pm), zl.shape[0], zp.shape[0],
        coef.shape[0], A, R, int(joint), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return (zl, zp, hl, hp) if joint else (zl, zp, hl)


SHAPES = {'configs2': ([25] * 64, [175] * 64), 'ragged': ([7, 1, 12, 3], [30, 0, 9, 140])}


@pytest.mark.parametrize('step', ['first', 'later'])
@pytest.mark.parametrize('shape', list(SHAPES))
@pytest.mark.parametrize('joint', [False, True], ids=['cond', 'joint'])
def test_multistep_kernel_against_float64(joint, shape, step):
    cfg = FULLATOM_JOINT if joint else FULLATOM_COND
    A, R = cfg.atom_nf, cfg.residue_nf
    n_lig, n_poc = SHAPES[shape]
    n = len(n_lig)
    g = torch.Generator(device='cuda').manual_seed(7)
    lm = torch.repeat_interleave(torch.arange(n, device='cuda'), torch.tensor(n_lig, device='cuda'))
    pm = torch.repeat_interleave(torch.arange(n, device='cuda'), torch.tensor(n_poc, device='cuda'))
    rnd = lambda r, c, s=1.0: torch.randn((r, c), device='cuda', generator=g) * s
    zl, zp = rnd(len(lm), 3 + A), rnd(len(pm), 3 + R, 4.0)
    eps_l, eps_p = rnd(len(lm), 3 + A), rnd(len(pm), 3 + R)
    hl, hp = rnd(len(lm), 3 + A, 2.0), rnd(len(pm), 3 + R, 2.0)
    ddpm = make_ddpm(FULLATOM_COND.with_(n_layers=1), False, timesteps=500)
    _, table = ddpm._fast_tables(N, 'dpmpp_2m', 0.0, 'cuda')
    rows = torch.tensor([N - 1 if step == 'first' else 20, 30, 5, 44], device='cuda')
    coef = table[rows[torch.arange(n, device='cuda') % 4]].contiguous()
    if step == 'first':
        coef[:, 4] = 0
        hl.fill_(float('nan')); hp.fill_(float('nan'))        # a first step never reads the history
    got = multistep(zl, zp, hl, hp, eps_l, eps_p, coef, lm, pm, A, R, joint)
    if step == 'first':
        hl.zero_(); hp.zero_()
    if joint:
        refs = [joint_multistep_ref(zl, zp, eps_l, eps_p, hl, hp, coef, lm, pm, d) for d in (torch.float32, torch.float64)]
        names = ('z_lig', 'z_pocket', 'hist_lig', 'hist_pocket')
    else:
        refs = [multistep_ref(zl, eps_l, hl, coef, zp, lm, pm, d) for d in (torch.float32, torch.float64)]
        refs = [(r[0], r[1], r[2]) for r in refs]
        names = ('z_lig', 'pocket', 'hist_lig')
    for k, name in enumerate(names):
        assert torch.isfinite(got[k]).all(), name
        assert_fp64_bound(got[k], refs[0][k], refs[1][k], f'{shape} {step} {name}')
    if not joint:
        assert torch.equal(got[1][:, 3:], zp[:, 3:]), 'the conditional pocket features must not change'
    again = multistep(zl, zp, hl, hp, eps_l, eps_p, coef, lm, pm, A, R, joint)
    assert all(torch.equal(a, b) for a, b in zip(got, again))
    # a graph's result does not depend on the rest of its batch: graph 1 alone
    l1, p1 = lm == 1, pm == 1
    one = multistep(zl[l1], zp[p1], hl[l1], hp[p1], eps_l[l1], eps_p[p1], coef[1:2].contiguous(), lm[l1] - 1, pm[p1] - 1,
                    A, R, joint)
    assert torch.equal(one[0], got[0][l1]) and torch.equal(one[1], got[1][p1]) and torch.equal(one[2], got[2][l1])


# ---- 2./3. teacher-forced graph engine ----------------------------------------------------------------------------------
def _record(ddpm, joint, sampler, eta, frames, seeds, inputs):
    """One seeded sampler call with the graph engine's fast loop replaced by a copy that records every replay."""
    rec = dict(step=[], z=[], pocket=[], hist=[], noise=[], t=[], coef=[], frames_at=[])
    zk, pk = ('zl', 'zp') if joint else ('z', 'pocket')
    name = '_graphed_joint_fast_loop' if joint else '_graphed_fast_loop'

    def loop(z_lig, z_pocket, lig_mask, pocket_mask, n_samples, timesteps, sampler_, eta_, return_frames, out_lig, out_pocket):
        dyn = ddpm.dynamics
        prev_defer, dyn.defer_status_check = dyn.defer_status_check, True
        if joint:
            st = ddpm._joint_engine(z_lig, z_pocket, lig_mask, pocket_mask, n_samples, timesteps, 1, sampler_, eta_)
            g = ddpm._joint_graph(st, sampler_, z_lig, z_pocket, timesteps - 1)
            ddpm._joint_start(st, z_lig, z_pocket, timesteps - 1)
        else:
            st = ddpm._engine(z_lig, z_pocket, lig_mask, pocket_mask, n_samples, timesteps, ddpm._seeds(), sampler_, eta_)
            g = ddpm._graph(st, sampler_, z_lig, z_pocket, timesteps - 1)
            ddpm._start(st, z_lig, z_pocket, timesteps - 1)
        hist = lambda: tuple(x.clone() for x in st['hist']) if joint else st['hist'].clone()
        for s in reversed(range(timesteps)):
            rec['step'].append(int(st['step'])); rec['z'].append(st[zk].clone()); rec['pocket'].append(st[pk].clone())
            rec['hist'].append(hist() if 'hist' in st else None)
            g.replay()
            rec['noise'].append(tuple(x.clone() for x in st['n_rev']) if joint else st['noise'].clone())
            rec['t'].append(st['t'].clone()); rec['coef'].append(st['coef_fast'].clone())
            if (s * return_frames) % timesteps == 0:
                idx = (s * return_frames) // timesteps
                out_lig[idx], out_pocket[idx] = ddpm.unnormalize_z(st[zk], st[pk])
                rec['frames_at'].append(s)
        dyn.defer_status_check = prev_defer
        dyn.check_status()
        rec['z'].append(st[zk].clone()); rec['pocket'].append(st[pk].clone())
        rec['hist'].append(hist() if 'hist' in st else None)
        rec['lm'], rec['pm'] = st['lig_mask'].clone(), st['pocket_mask'].clone()
        return st[zk].clone(), st[pk].clone()

    setattr(ddpm, name, loop)
    try:
        rec['out'] = _call(ddpm, joint, inputs, seeds, frames=frames, timesteps=N, sampler=sampler, eta=eta)
    finally:
        delattr(ddpm, name)
    return rec


def _call(ddpm, joint, inputs, seeds, **kw):
    if joint:
        n_lig, n_poc = inputs
        return ddpm.sample(len(n_lig), n_lig, n_poc, return_frames=kw.pop('frames', 1), device='cuda', seeds=seeds, **kw)
    pocket, n_lig = inputs
    return ddpm.sample_given_pocket({k: v.clone() for k, v in pocket.items()}, n_lig, return_frames=kw.pop('frames', 1),
                                    seeds=seeds, **kw)


@pytest.fixture(scope='module', params=['cond', 'joint'])
def model(request):
    joint = request.param == 'joint'
    ddpm = make_ddpm(FULLATOM_JOINT if joint else FULLATOM_COND, joint, timesteps=500)
    if joint:
        inputs = (torch.tensor(JOINT_LIG).cuda(), torch.tensor(JOINT_POC).cuda())
    else:
        inputs = full_pocket()
    seeds = torch.arange(500, 500 + len(inputs[1]))
    return joint, ddpm, inputs, seeds


@pytest.mark.parametrize('sampler,eta', RUNS + [('ddim', 1.0)])
def test_graph_engine_teacher_forced(model, sampler, eta):
    joint, ddpm, inputs, seeds = model
    frames = 5
    rec = _record(ddpm, joint, sampler, eta, frames, seeds, inputs)
    dyn, lm, pm = ddpm.dynamics, rec['lm'], rec['pm']
    n = rec['t'][0].shape[0]
    t_table, table = ddpm._fast_tables(N, sampler, eta, 'cuda')
    assert rec['step'] == list(range(N - 1, -1, -1))
    assert rec['frames_at'] == [s for s in range(N - 1, -1, -1) if s % (N // frames) == 0]
    if eta == 1.0:
        _, anc = ddpm._joint_tables(N, 1, 'cuda') if joint else ddpm._schedule_tables(N, N, 'cuda')
    for k, s in enumerate(rec['step']):
        c = rec['coef'][k]
        assert torch.equal(c, table[s].expand_as(c)) and torch.equal(rec['t'][k], t_table[s].expand(n, 1))
        z, p, h = rec['z'][k], rec['pocket'][k], rec['hist'][k]
        with torch.no_grad():
            eps_l, eps_p = dyn(z, p, rec['t'][k], lm, pm)
        noise = rec['noise'][k] if eta > 0 else None
        if eta > 0:       # the ancestral step's draw id (STAGE_LOOP, s, 0, PURPOSE_REVERSE)
            did = torch.full((1,), seeded.draw_id(seeded.STAGE_LOOP, s, 0, seeded.PURPOSE_REVERSE), dtype=torch.int64,
                             device='cuda')
            sd = seeds.cuda()
            if joint:
                want = [seeded.fill(torch.empty_like(x), r, sd, did, lm, pm)
                        for x, r in zip(noise, (_native.RNG_JOINT_X, _native.RNG_LIGAND, _native.RNG_POCKET))]
                assert all(torch.equal(a, b) for a, b in zip(noise, want))
            else:
                assert torch.equal(noise, seeded.fill(torch.empty_like(noise), _native.RNG_LIGAND, sd, did, lm, pm))
        else:
            assert all(not x.any() for x in (rec['noise'][k] if joint else (rec['noise'][k],))), 'eta = 0 draws nothing'
        if sampler == 'ddim' and joint:
            refs = [joint_ddim_ref(z, p, eps_l, eps_p, noise, c, lm, pm, d) for d in (torch.float32, torch.float64)]
            got = (rec['z'][k + 1], rec['pocket'][k + 1])
        elif sampler == 'ddim':
            refs = [ddim_ref(z, eps_l, noise, c, p, lm, pm, d) for d in (torch.float32, torch.float64)]
            got = (rec['z'][k + 1], rec['pocket'][k + 1])
        elif joint:
            refs = [joint_multistep_ref(z, p, eps_l, eps_p, h[0], h[1], c, lm, pm, d) for d in (torch.float32, torch.float64)]
            got = (rec['z'][k + 1], rec['pocket'][k + 1]) + rec['hist'][k + 1]
        else:
            refs = [multistep_ref(z, eps_l, h, c, p, lm, pm, d) for d in (torch.float32, torch.float64)]
            got = (rec['z'][k + 1], rec['pocket'][k + 1], rec['hist'][k + 1])
        for i, x in enumerate(got):
            assert_fp64_bound(x, refs[0][i], refs[1][i], f'{sampler} eta={eta} s={s} output {i}')
        if eta == 1.0:    # the ancestral step on the same state and noise, with its own fp32 coefficients
            ca = anc[s, :3].expand(n, 3).contiguous()
            if joint:
                anc_got = joint_update(ddpm, z, p, eps_l, eps_p, noise, ca, lm, pm)
                a32 = joint_ddim_ref(z, p, eps_l, eps_p, noise, ca, lm, pm, torch.float32)
            else:
                anc_got = ligand_update(ddpm, z, eps_l, noise, ca, p, lm, pm)
                a32 = ddim_ref(z, eps_l, noise, ca, p, lm, pm, torch.float32)
            for i in range(2):
                assert_fp64_bound(anc_got[i], a32[i], refs[1][i], f'ddpm step s={s} output {i} vs float64 DDIM(eta=1)')
    assert torch.isfinite(rec['z'][-1]).all()


# ---- 4. regeneration, re-capture, the default ---------------------------------------------------------------------------
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


def _rows(out, mask, g, frames):
    return out[:, mask == g] if frames > 1 else out[mask == g]


@pytest.mark.parametrize('engine', ['graph', 'eager'])
@pytest.mark.parametrize('sampler,eta', RUNS)
@pytest.mark.parametrize('joint', [False, True], ids=['cond', 'joint'])
def test_regenerate_graphs_alone_and_reversed(joint, sampler, eta, engine):
    frames = 5
    _, run = _runner(joint, engine, frames, sampler=sampler, eta=eta, timesteps=N)
    full = run(list(range(64)))
    assert torch.isfinite(full[0]).all()
    for idx in ([0], [37], [63], [63, 37, 0]):
        sub = run(idx)
        for k, g in enumerate(idx):
            for part, mi in ((0, 2), (1, 3)):
                assert torch.equal(_rows(sub[part], sub[mi], k, frames), _rows(full[part], full[mi], g, frames)), \
                    (sampler, eta, engine, idx, g, part)


@pytest.mark.parametrize('joint', [False, True], ids=['cond', 'joint'])
def test_sampler_switch_recaptures_and_default_is_ddpm(joint):
    ddpm, run = _runner(joint, 'graph', 1, timesteps=N)
    cache = lambda: ddpm._joint_cache if joint else ddpm._graph_cache
    idx = list(range(64))
    a = run(idx, sampler='ddim')
    st_a = next(iter(cache().values()))
    b = run(idx, sampler='dpmpp_2m')
    st_b = next(iter(cache().values()))
    assert st_b is not st_a and 'dpmpp_2m' in st_b['graphs'] and len(cache()) == 1
    c = run(idx, sampler='ddim')
    assert next(iter(cache().values())) is not st_b
    assert all(torch.equal(x, y) for x, y in zip(a, c)), 'switching back to ddim changed the bits'
    assert not torch.equal(a[0], b[0])
    d, e = run(idx), run(idx, sampler='ddpm')
    assert all(torch.equal(x, y) for x, y in zip(d, e)), "sampler='ddpm' differs from the default call"
    assert not torch.equal(a[0], d[0])


# ---- 5. NaN status ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('engine', ['graph', 'eager'])
@pytest.mark.parametrize('sampler', ['ddpm', 'ddim', 'dpmpp_2m'])
def test_nan_reports_as_for_the_ancestral_sampler(sampler, engine):
    ddpm, cfg = _small(False, engine)
    pocket = {k: v.cuda() for k, v in syn.synthetic_pocket(cfg, [20, 14], seed=2, spread=3.0).items()}
    bad = {k: v.clone() for k, v in pocket.items()}
    bad['one_hot'] = bad['one_hot'].float()
    bad['one_hot'][3, 1] = float('nan')
    n_lig = torch.tensor([5, 4]).cuda()
    with pytest.raises(ValueError, match='NaN detected in EGNN output'):
        ddpm.sample_given_pocket(bad, n_lig, timesteps=10, sampler=sampler)
    out = ddpm.sample_given_pocket(pocket, n_lig, timesteps=10, sampler=sampler)     # the sticky flag was cleared
    assert torch.isfinite(out[0]).all()
