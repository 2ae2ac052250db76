"""CPU: few-step RePaint inpainting and diversify (DESIGN §14) against float64 and against the ancestral sampler.

1. Anchors, on a cut-off-free model with the float64 oracle denoiser and one torch seed: DDIM at eta = 1 reproduces the
   ancestral conditional inpaint, joint inpaint and diversify within the fp32 rounding of its coefficient table.
2. Each eager fp32 RePaint round against its float64 restatement (fast_repaint_cases), both models, DDIM at eta 0 / 0.5 / 1
   and 2M, on re-noised rounds that do not commit and on the last round of a step, which commits; on a round that does not
   commit the 2M history keeps its offset to the pocket (conditional) or is only translated, one shift per graph (joint).
3. 2M diversify on the t* grid is second order, DDIM first order.
4. Every refusal happens before any draw; explicit sampler='ddpm' is the default call, bit for bit.
"""
import math

import pytest
import torch

from ddpm_cases import DDPM_CFG, HIST, JOINT_CFG, assert_fp64_bound, make_ligand, make_pocket
from fast_repaint_cases import cond_round_ref, joint_round_ref
from diffsbdd_b200 import synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM, SimpleConditionalDDPM
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion, fast_coefficients, scatter_mean
from oracle import egnn_oracle
from oracle.cpu_denoiser import OracleDynamics

FREE = dict(edge_cutoff_pocket=None, edge_cutoff_interaction=None)      # continuous field (DESIGN §5)


class _Oracle64(torch.nn.Module):
    """The float64 oracle denoiser behind the fp32 sampler interface."""

    def __init__(self, cfg, seed):
        super().__init__()
        self.cfg, self.sd = cfg, syn.synthetic_state_dict(cfg, seed)
        self.update_pocket_coords = cfg.update_pocket_coords

    def forward(self, xa, xr, t, ma, mr):
        out = egnn_oracle.denoiser_forward(self.cfg, self.sd, xa.double(), xr.double(), t.double(), ma, mr, dtype=torch.float64)
        return tuple(x.float() for x in out)


class _Recording(torch.nn.Module):
    def __init__(self, inner):
        super().__init__()
        self.inner, self.out = inner, None
        self.update_pocket_coords = inner.update_pocket_coords

    def forward(self, *args):
        self.out = self.inner(*args)
        return self.out


def _ddpm(cfg=DDPM_CFG, joint=False, T=20, dynamics=None, cls=None):
    cls = cls or (EnVariationalDiffusion if joint else ConditionalDDPM)
    dyn = dynamics if dynamics is not None else OracleDynamics(cfg, syn.synthetic_state_dict(cfg, 5))
    return cls(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=T,
               noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2', norm_values=(1, 4),
               size_histogram=HIST).eval()


def _inputs(n_lig=(7, 5), n_fixed=3):
    ligand, fixed = make_ligand(list(n_lig), n_fixed)
    return ligand, make_pocket(), fixed


def _copy(d):
    return {k: v.clone() for k, v in d.items()}


def _joint_fixed(pocket):
    f = torch.ones(len(pocket['mask']))
    f[::4] = 0                                  # a partly free pocket exercises the pocket blend
    return f


def _assert_anchor(a, b, what):
    """DDIM(eta = 1) against the ancestral sampler: the same formulas up to the fp32 rounding of the coefficient table (half
    an ulp against the ancestral ops' own fp32 error), carried through the trajectory; 2^-14 of the output's magnitude is
    about 500 fp32 ulp."""
    for k, (x, y) in enumerate(zip(a, b)):
        if x.dtype.is_floating_point:
            err, big = float((x - y).abs().max()), float(y.abs().max())
            assert err <= 2.0 ** -14 * max(big, 1.0), f'{what} output {k}: |DDIM(eta=1) - ancestral| = {err:.3e} (max {big:.3e})'
        else:
            assert torch.equal(x, y), f'{what} output {k}'


# ---- 1. anchors --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('resamplings', [1, 3])
def test_conditional_inpaint_ddim_eta1_is_ancestral(resamplings):
    cfg = DDPM_CFG.with_(**FREE)
    ddpm = _ddpm(cfg, T=8, dynamics=_Oracle64(cfg, 11))
    ligand, pocket, fixed = _inputs()
    outs = []
    for kw in ({}, dict(sampler='ddim', eta=1.0)):
        torch.manual_seed(21)
        outs.append(ddpm.inpaint(_copy(ligand), _copy(pocket), fixed, resamplings=resamplings, **kw))
    _assert_anchor(outs[1], outs[0], f'conditional inpaint r={resamplings}')


@pytest.mark.parametrize('jump_length', [1, 2])
def test_joint_inpaint_ddim_eta1_is_ancestral(jump_length):
    cfg = JOINT_CFG.with_(**FREE)
    ddpm = _ddpm(cfg, joint=True, T=8, dynamics=_Oracle64(cfg, 12))
    ligand, pocket, fixed = _inputs(n_fixed=2)
    outs = []
    for kw in ({}, dict(sampler='ddim', eta=1.0)):
        torch.manual_seed(22)
        outs.append(ddpm.inpaint(_copy(ligand), _copy(pocket), fixed, _joint_fixed(pocket), resamplings=2,
                                 jump_length=jump_length, **kw))
    _assert_anchor(outs[1], outs[0], f'joint inpaint j={jump_length}')


def test_diversify_ddim_eta1_is_ancestral():
    cfg = DDPM_CFG.with_(**FREE)
    ddpm = _ddpm(cfg, T=12, dynamics=_Oracle64(cfg, 13))
    ligand, pocket, _ = _inputs()
    outs = []
    for kw in ({}, dict(sampler='ddim', eta=1.0, denoising_steps=6)):
        torch.manual_seed(23)
        outs.append(ddpm.diversify(_copy(ligand), _copy(pocket), 6, **kw))
    _assert_anchor(outs[1], outs[0], 'diversify')


# ---- 2. eager rounds against float64 -----------------------------------------------------------------------------------
RUNS = [('ddim', 0.0), ('ddim', 0.5), ('ddim', 1.0), ('dpmpp_2m', 0.0)]
N_STEPS, ROUNDS = 5, 2


def _offsets(h, p, lm, pm):
    """Per graph: COM of the history's coordinates minus COM of the pocket's (the offset a translation of both keeps)."""
    return scatter_mean(h[:, :3].double(), lm) - scatter_mean(p[:, :3].double(), pm)


@pytest.mark.parametrize('sampler,eta', RUNS)
def test_eager_conditional_rounds_against_float64(sampler, eta):
    torch.manual_seed(3)
    ddpm = _ddpm()
    ddpm.dynamics = rec = _Recording(ddpm.dynamics)
    ligand, pocket, fixed = _inputs()
    ligand, pocket = ddpm.normalize(ligand, pocket)
    lm, pm = ligand['mask'], pocket['mask']
    xh_pocket = torch.cat([pocket['x'], pocket['one_hot']], 1)
    xh_ligand = torch.cat([ligand['x'], ligand['one_hot']], 1)
    com0 = scatter_mean(pocket['x'], pm, dim=0)
    z = torch.randn(len(lm), 3 + DDPM_CFG.atom_nf)
    z[:, :3], xh_pocket[:, :3] = ddpm.remove_mean_batch(z[:, :3], xh_pocket[:, :3], lm, pm)
    hist = ddpm._empty_history(z, sampler)
    t_table, coef = ddpm._fast_tables(N_STEPS, sampler, eta, 'cpu')
    _, anc = ddpm._schedule_tables(N_STEPS, N_STEPS, 'cpu')
    noises = []
    lig_noise = ddpm._lig_noise
    ddpm._lig_noise = lambda *a: noises.append(lig_noise(*a)) or noises[-1]
    for s in reversed(range(N_STEPS)):
        sa = torch.full((2, 1), float(s))
        for u in range(ROUNDS):
            last = u == ROUNDS - 1
            noises.clear()
            out = ddpm._fast_inpaint_step(s, u, t_table[s].expand(2, 1), coef[s:s + 1], ddpm.gamma(sa / N_STEPS),
                                          ddpm.gamma((sa + 1) / N_STEPS), z, xh_pocket, hist, ligand['x'], xh_ligand.clone(),
                                          com0, fixed.view(-1, 1), lm, pm, sampler, eta, last)
            k = int(sampler == 'ddim' and eta > 0)
            assert len(noises) == k + 1 + (not last), 'draws: reverse (DDIM, eta > 0), known part, re-noise'
            h = hist[0] if hist else torch.zeros_like(z)
            args = (z, xh_pocket, h, rec.out[0], noises[0] if k else None, noises[k], None if last else noises[k + 1],
                    coef[s:s + 1].expand(2, -1), anc[s:s + 1, 3:].expand(2, -1), xh_ligand, com0, fixed, lm, pm, sampler, last)
            refs = [cond_round_ref(*args, d) for d in (torch.float32, torch.float64)]
            got = out[:2] + out[2]
            assert len(got) == (3 if sampler == 'dpmpp_2m' else 2)
            for i, name in enumerate(('z', 'pocket', 'hist')[:len(got)]):
                assert_fp64_bound(got[i], refs[0][i], refs[1][i], f'{sampler} eta={eta} s={s} u={u} {name}')
            if sampler == 'dpmpp_2m' and not last:
                before, after = _offsets(h, xh_pocket, lm, pm), _offsets(out[2][0], out[1], lm, pm)
                assert float((after - before).abs().max()) <= 1e-5, 'a round that does not commit moved hist against the pocket'
            z, xh_pocket, hist = out


@pytest.mark.parametrize('sampler,eta', RUNS)
def test_eager_joint_rounds_against_float64(sampler, eta):
    torch.manual_seed(4)
    ddpm = _ddpm(JOINT_CFG, joint=True)
    ddpm.dynamics = rec = _Recording(ddpm.dynamics)
    ligand, pocket, fixed = _inputs(n_fixed=2)
    ligand, pocket = ddpm.normalize(ligand, pocket)
    lm, pm = ligand['mask'], pocket['mask']
    fp = _joint_fixed(pocket)
    xl, xp = torch.cat([ligand['x'], ligand['one_hot']], 1), torch.cat([pocket['x'], pocket['one_hot']], 1)
    zl, zp = ddpm.sample_combined_position_feature_noise(lm, pm)
    hist = ((torch.zeros_like(zl),), (torch.zeros_like(zp),)) if sampler == 'dpmpp_2m' else ()
    t_table, coef = ddpm._fast_tables(N_STEPS, sampler, eta, 'cpu')
    _, anc = ddpm._joint_tables(N_STEPS, 1, 'cpu')
    noises = []
    draw = ddpm.sample_combined_position_feature_noise
    ddpm.sample_combined_position_feature_noise = lambda *a: noises.append(draw(*a)) or noises[-1]
    as_kernel = lambda e: (torch.cat((e[0][:, :3], e[1][:, :3])), e[0][:, 3:], e[1][:, 3:])
    lsel, psel = fixed.bool(), fp.bool()
    for s in reversed(range(N_STEPS)):
        sa = torch.full((2, 1), float(s))
        for u in range(ROUNDS):
            commit = u == ROUNDS - 1
            noises.clear()
            gs = ddpm.gamma(sa / N_STEPS)
            zl1, zp1, h1 = ddpm._joint_fast_inpaint_step(s, 0, t_table[s].expand(2, 1), coef[s:s + 1], gs, zl, zp, hist, xl, xp,
                                                         fixed.view(-1, 1), fp.view(-1, 1), lsel, psel, lm, pm, sampler, eta,
                                                         commit)
            if not commit:
                zl1, zp1, h1 = ddpm._joint_renoise(zl1, zp1, h1, ddpm.gamma((sa + 1) / N_STEPS), gs, lm, pm)
            k = int(sampler == 'ddim' and eta > 0)
            assert len(noises) == k + 1 + (not commit), 'draws: known part, reverse (DDIM, eta > 0), jump back'
            hl, hp = (hist[0][0], hist[1][0]) if hist else (torch.zeros_like(zl), torch.zeros_like(zp))
            args = (zl, zp, hl, hp, rec.out[0], rec.out[1], as_kernel(noises[1]) if k else None, as_kernel(noises[0]),
                    None if commit else as_kernel(noises[k + 1]), coef[s:s + 1].expand(2, -1), anc[s:s + 1, 3:].expand(2, -1),
                    xl, xp, fixed, fp, lm, pm, sampler, commit)
            refs = [joint_round_ref(*args, d) for d in (torch.float32, torch.float64)]
            got = (zl1, zp1) + sum(h1, ())
            for i, name in enumerate(('z_lig', 'z_pocket', 'hist_lig', 'hist_pocket')[:len(got)]):
                assert_fp64_bound(got[i], refs[0][i], refs[1][i], f'{sampler} eta={eta} s={s} u={u} {name}')
            if sampler == 'dpmpp_2m' and not commit:    # the history is only translated, one shift per graph for all its nodes
                move = torch.cat((h1[0][0][:, :3] - hl[:, :3], h1[1][0][:, :3] - hp[:, :3])).double()
                cm = torch.cat((lm, pm))
                assert float((move - scatter_mean(move, cm)[cm]).abs().max()) <= 1e-5
                assert torch.equal(h1[0][0][:, 3:], hl[:, 3:]) and torch.equal(h1[1][0][:, 3:], hp[:, 3:])
            zl, zp, hist = zl1, zp1, h1


# ---- 3. convergence order of diversify on the t* grid -----------------------------------------------------------------
T_ORDER, NOISING = 3200, 1600
K_ORDER = (25, 50, 100, 200, 400)


def _solve(ddpm, den, z, pocket, lm, pm, K, sampler):
    """diversify's reverse loop in float64 from t* = NOISING / T_ORDER: the grid of _fast_tables, fast_coefficients on it."""
    from fast_sampler_cases import ddim_ref, multistep_ref
    t_arr, _ = ddpm._fast_tables(K, sampler, 0.0, 'cpu', (NOISING, T_ORDER))
    s_arr = torch.cat((torch.zeros(1, 1), t_arr[:-1]))
    coef = fast_coefficients(ddpm.gamma(s_arr), ddpm.gamma(t_arr), sampler, 0.0)
    hist = torch.zeros_like(z)
    for s in reversed(range(K)):
        c = coef[s:s + 1].expand(2, -1)
        eps = den(z, pocket, t_arr[s].double().expand(2, 1), lm, pm)
        if sampler == 'ddim':
            z, pocket = ddim_ref(z, eps, None, c, pocket, lm, pm, torch.float64)
        else:
            z, pocket, hist = multistep_ref(z, eps, hist, c, pocket, lm, pm, torch.float64)
    return z


@pytest.mark.timeout(900)
def test_diversify_convergence_order():
    cfg = DDPM_CFG.with_(**FREE)
    sd = syn.synthetic_state_dict(cfg, 11)
    ddpm = _ddpm(cfg, T=T_ORDER)

    def den(z, pocket, t, lm, pm):
        return egnn_oracle.denoiser_forward(cfg, sd, z, pocket, t, lm, pm, dtype=torch.float64)[0]

    g = torch.Generator().manual_seed(6)
    n_lig, n_poc = [5, 4], [8, 6]
    lm, pm = torch.repeat_interleave(torch.arange(2), torch.tensor(n_lig)), torch.repeat_interleave(torch.arange(2), torch.tensor(n_poc))
    # a partially noised ligand at t* = 1/2: data-scale coordinates plus noise
    z = torch.randn((sum(n_lig), 3 + cfg.atom_nf), generator=g, dtype=torch.float64)
    pocket = torch.cat([torch.randn((sum(n_poc), 3), generator=g, dtype=torch.float64) * 1.5,
                        torch.nn.functional.one_hot(torch.arange(sum(n_poc)) % cfg.residue_nf, cfg.residue_nf).double() / 4], 1)
    z[:, :3], pocket[:, :3] = ddpm.remove_mean_batch(z[:, :3], pocket[:, :3], lm, pm)
    ref = _solve(ddpm, den, z, pocket, lm, pm, NOISING, 'dpmpp_2m')
    orders = {}
    for sampler in ('ddim', 'dpmpp_2m'):
        err = [float((_solve(ddpm, den, z, pocket, lm, pm, K, sampler) - ref).abs().max()) for K in K_ORDER]
        orders[sampler] = [math.log2(a / b) for a, b in zip(err, err[1:])]
        print(sampler, ['%.3e' % e for e in err], ['%.3f' % o for o in orders[sampler]])
    assert 0.8 <= orders['ddim'][-1] <= 1.2, f"DDIM observed order {orders['ddim']}"
    assert orders['dpmpp_2m'][-1] >= 1.7, f"DPM-Solver++(2M) observed order {orders['dpmpp_2m']}"


# ---- 4. refusals before any draw, and the default ----------------------------------------------------------------------
def _refused(call):
    state = torch.random.get_rng_state()
    with pytest.raises(ValueError):
        call()
    assert torch.equal(state, torch.random.get_rng_state()), 'a draw happened before the arguments were refused'


@pytest.mark.parametrize('sampler,eta', [('euler', 0.0), ('ddim', 1.5), ('dpmpp_2m', 0.3), ('ddpm', 0.5)])
def test_invalid_sampler_arguments_raise_before_any_draw(sampler, eta):
    cond, joint = _ddpm(), _ddpm(JOINT_CFG, joint=True)
    ligand, pocket, fixed = _inputs()
    _refused(lambda: cond.inpaint(_copy(ligand), _copy(pocket), fixed, sampler=sampler, eta=eta))
    _refused(lambda: cond.diversify(_copy(ligand), _copy(pocket), 5, sampler=sampler, eta=eta))
    _refused(lambda: joint.inpaint(_copy(ligand), _copy(pocket), fixed, torch.ones(len(pocket['mask'])), sampler=sampler,
                                   eta=eta))


def test_specific_refusals_before_any_draw():
    cond, joint = _ddpm(), _ddpm(JOINT_CFG, joint=True)
    simple = _ddpm(cls=SimpleConditionalDDPM)
    ligand, pocket, fixed = _inputs()
    pf = torch.ones(len(pocket['mask']))
    _refused(lambda: joint.inpaint(_copy(ligand), _copy(pocket), fixed, pf, resamplings=2, jump_length=2, sampler='dpmpp_2m'))
    for sampler in ('ddim', 'dpmpp_2m'):
        _refused(lambda: simple.inpaint(_copy(ligand), _copy(pocket), fixed, sampler=sampler))
        _refused(lambda: simple.diversify(_copy(ligand), _copy(pocket), 5, sampler=sampler))
        _refused(lambda: cond.diversify(_copy(ligand), _copy(pocket), 5, sampler=sampler, denoising_steps=0))
        _refused(lambda: cond.diversify(_copy(ligand), _copy(pocket), 5, sampler=sampler, denoising_steps=6))
    _refused(lambda: cond.diversify(_copy(ligand), _copy(pocket), 5, denoising_steps=3))
    _refused(lambda: cond.diversify(_copy(ligand), _copy(pocket), 5, sampler='ddpm', denoising_steps=0))
    # joint DDIM may jump over several steps
    joint.inpaint(_copy(ligand), _copy(pocket), fixed, pf, resamplings=2, jump_length=2, sampler='ddim', timesteps=4)


def test_explicit_ddpm_is_the_default_call():
    cond, joint = _ddpm(T=6), _ddpm(JOINT_CFG, joint=True, T=6)
    ligand, pocket, fixed = _inputs()
    pf = _joint_fixed(pocket)
    calls = [
        lambda **kw: cond.inpaint(_copy(ligand), _copy(pocket), fixed, resamplings=2, **kw),
        lambda **kw: cond.diversify(_copy(ligand), _copy(pocket), 4, **kw),
        lambda **kw: joint.inpaint(_copy(ligand), _copy(pocket), fixed, pf, resamplings=2, jump_length=2, **kw),
    ]
    for k, call in enumerate(calls):
        outs = []
        for kw in ({}, dict(sampler='ddpm', eta=0.0), dict(sampler='ddpm', denoising_steps=4) if k == 1 else {}):
            torch.manual_seed(30 + k)
            outs.append(call(**kw))
        for o in outs[1:]:
            assert all(torch.equal(a, b) for a, b in zip(outs[0], o)), f"call {k}: sampler='ddpm' differs from the default"

