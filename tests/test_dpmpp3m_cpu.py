"""CPU: the third-order multistep sampler 'dpmpp_3m' (DESIGN §15) against float64, without a GPU.

1. Coefficient tables: each fp32 row within half an ulp of the exact D1 / D2 form (mpmath from the same fp32 gammas) for the
   polynomial, cosine and learned schedules at N in {T, T/5, T/50}; k0 + k1 + k2 = -alpha_s phi1; the first row run is DDIM
   at eta = 0 and the second is 2M's.
2. One eager fp32 step of each model and one RePaint round of each model against their float64 restatements
   (dpmpp3m_cases), along short trajectories that cover the first, the second and later steps.
3. Convergence on the cut-off-free float64 oracle set-up of §13: observed orders of 2M and 3M; 3M closer to the converged
   solution than 2M from N = 100 up, and an observed order of at least 2.25 over the two finest halvings.
4. Refusals before any draw.
"""
import math

import pytest
import torch

from ddpm_cases import DDPM_CFG, HIST, JOINT_CFG, assert_fp64_bound, make_ligand, make_pocket
from dpmpp3m_cases import (closed_form_rows, cond_round3_ref, joint_multistep3_ref, joint_round3_ref, multistep3_ref)
from diffsbdd_b200 import synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM, SimpleConditionalDDPM
from diffsbdd_b200.distributed import sample_given_pocket_sharded
from diffsbdd_b200.en_diffusion import (EnVariationalDiffusion, check_sampler, fast_coefficients, num_nodes_to_batch_mask,
                                        scatter_mean)
from oracle import egnn_oracle
from oracle.cpu_denoiser import OracleDynamics

SCHEDULES = ('polynomial_2', 'cosine', 'learned')
T_TABLE = 500


def _ddpm(cfg=DDPM_CFG, joint=False, T=20, schedule='polynomial_2', cls=None):
    cls = cls or (EnVariationalDiffusion if joint else ConditionalDDPM)
    dyn = OracleDynamics(cfg, syn.synthetic_state_dict(cfg, 5))
    return cls(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=T, noise_schedule=schedule,
               noise_precision=5e-4, loss_type='vlb' if schedule == 'learned' else 'l2', norm_values=(1, 4),
               size_histogram=HIST).eval()


def _gammas(ddpm, N):
    s_int = torch.arange(N).view(-1, 1)
    return ddpm.gamma(s_int / N).detach(), ddpm.gamma((s_int + 1) / N).detach()


# ---- 1. coefficient tables ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('schedule', SCHEDULES)
@pytest.mark.parametrize('N', [T_TABLE, T_TABLE // 5, T_TABLE // 50])
def test_3m_table_is_the_closed_form_rounded(schedule, N):
    torch.manual_seed(0)
    ddpm = _ddpm(T=T_TABLE, schedule=schedule)
    gs, gt = _gammas(ddpm, N)
    exact = closed_form_rows(gs, gt)
    _, fast = ddpm._fast_tables(N, 'dpmpp_3m', 0.0, 'cpu')
    assert fast.shape == (N, 6) and fast.dtype == torch.float32
    worst = 0.0
    for k in range(N):
        for j in range(6):
            e = exact[k][j]
            if e == 0:
                assert fast[k, j] == 0, f'{schedule} N={N} row {k} col {j}: {float(fast[k, j])} for an exact 0'
                continue
            ulp = 2.0 ** (math.floor(math.log2(abs(float(e)))) - 23)
            worst = max(worst, abs(float(fast[k, j]) - float(e)) / ulp)
    # the float64 evaluation is exact to ~1e-15 relative, so a value within that of a rounding midpoint may round either way
    assert worst <= 0.5 + 1e-6, f'{schedule} N={N}: fp32 row off the closed form by {worst:.4f} ulp'
    c64 = fast_coefficients(gs, gt, 'dpmpp_3m')
    c1 = -torch.sqrt(torch.sigmoid(-gs.double())) * torch.expm1(-0.5 * (gt.double() - gs.double()))
    rel = ((c64[:, 3:].sum(1, keepdim=True) - c1).abs() / c1.abs()).max()
    assert rel <= 1e-12, f'{schedule} N={N}: k0 + k1 + k2 != -alpha_s phi1 (relative {rel:.2e})'
    if N >= 3:
        assert bool((c64[:-2, 5] > 0).all()), 'every third-order row reads m2'


@pytest.mark.parametrize('schedule', SCHEDULES)
def test_first_3m_row_is_ddim_eta0_and_second_is_2m(schedule):
    torch.manual_seed(0)
    ddpm = _ddpm(T=T_TABLE, schedule=schedule)
    gs, gt = _gammas(ddpm, T_TABLE // 5)
    m3, m2, ddim = (fast_coefficients(gs, gt, s, 0.0) for s in ('dpmpp_3m', 'dpmpp_2m', 'ddim'))
    first, second = m3[-1], m3[-2]
    assert first[4] == 0 and first[5] == 0 and second[5] == 0 and second[4] != 0
    z, eps = torch.randn(50, dtype=torch.float64), torch.randn(50, dtype=torch.float64)
    a = z / ddim[-1, 0] - ddim[-1, 1] * eps
    b = first[0] * z + first[3] * ((z - first[2] * eps) * first[1])
    assert float((a - b).abs().max()) <= 1e-12 * float(a.abs().max())
    # the second row is 2M's second step: the same (c0, 1/alpha_t, sigma_t) and k0 = c1 (1 + w), k1 = -c1 w
    c1, w = m2[-2, 1], m2[-2, 4]
    assert second[0] == m2[-2, 0] and second[1] == m2[-2, 2] and second[2] == m2[-2, 3]
    assert second[3] == c1 * (1 + w) and second[4] == -c1 * w


def test_n1_and_n2_grids():
    ddpm = _ddpm(T=T_TABLE)
    for N in (1, 2):
        _, fast = ddpm._fast_tables(N, 'dpmpp_3m', 0.0, 'cpu')
        assert fast.shape == (N, 6) and bool(torch.isfinite(fast).all())
        assert fast[-1, 4] == 0 and fast[-1, 5] == 0 and fast[0, 5] == 0
    torch.manual_seed(1)
    out = ddpm.sample_given_pocket(make_pocket(), torch.tensor([5, 6]), timesteps=2, sampler='dpmpp_3m')
    assert bool(torch.isfinite(out[0]).all())


# ---- 2. the eager engine, teacher-forced -------------------------------------------------------------------------------
class _Recording(torch.nn.Module):
    """The denoiser, keeping its last output."""

    def __init__(self, inner):
        super().__init__()
        self.inner, self.out = inner, None
        self.update_pocket_coords = inner.update_pocket_coords

    def forward(self, *args):
        self.out = self.inner(*args)
        return self.out


N_STEPS = 6


def test_eager_conditional_steps_against_float64():
    torch.manual_seed(3)
    ddpm = _ddpm()
    ddpm.dynamics = rec = _Recording(ddpm.dynamics)
    _, pocket = ddpm.normalize(pocket=make_pocket())
    lm, pm = num_nodes_to_batch_mask(2, torch.tensor([7, 5]), 'cpu'), pocket['mask']
    xh_pocket = torch.cat([pocket['x'], pocket['one_hot']], 1)
    z = torch.randn(12, 3 + DDPM_CFG.atom_nf)
    z[:, :3], xh_pocket[:, :3] = ddpm.remove_mean_batch(z[:, :3], xh_pocket[:, :3], lm, pm)
    hist = ddpm._empty_history(z, 'dpmpp_3m')
    t_table, coef = ddpm._fast_tables(N_STEPS, 'dpmpp_3m', 0.0, 'cpu')
    for s in reversed(range(N_STEPS)):
        z1, p1, h1 = ddpm._fast_step(s, t_table[s].expand(2, 1), coef[s:s + 1], z, xh_pocket, hist, lm, pm, 'dpmpp_3m', 0.0)
        c = coef[s:s + 1].expand(2, -1)
        refs = [multistep3_ref(z, rec.out[0], *hist, c, xh_pocket, lm, pm, d) for d in (torch.float32, torch.float64)]
        for k, (name, got) in enumerate(zip(('z', 'pocket', 'm1', 'm2'), (z1, p1) + tuple(h1))):
            assert_fp64_bound(got, refs[0][k], refs[1][k], f'3M s={s} {name}')
        z, xh_pocket, hist = z1, p1, h1


def test_eager_joint_steps_against_float64():
    torch.manual_seed(4)
    ddpm = _ddpm(JOINT_CFG, joint=True)
    ddpm.dynamics = rec = _Recording(ddpm.dynamics)
    lm = num_nodes_to_batch_mask(2, torch.tensor([6, 4]), 'cpu')
    pm = num_nodes_to_batch_mask(2, torch.tensor([9, 12]), 'cpu')
    zl, zp = ddpm.sample_combined_position_feature_noise(lm, pm)
    hl, hp = ddpm._empty_history(zl, 'dpmpp_3m'), ddpm._empty_history(zp, 'dpmpp_3m')
    t_table, coef = ddpm._fast_tables(N_STEPS, 'dpmpp_3m', 0.0, 'cpu')
    for s in reversed(range(N_STEPS)):
        out = ddpm._joint_fast_step(s, t_table[s].expand(2, 1), coef[s:s + 1], zl, zp, hl, hp, lm, pm, 'dpmpp_3m', 0.0)
        c = coef[s:s + 1].expand(2, -1)
        refs = [joint_multistep3_ref(zl, zp, *rec.out, hl[0], hp[0], hl[1], hp[1], c, lm, pm, d)
                for d in (torch.float32, torch.float64)]
        got = (out[0], out[1], out[2][0], out[3][0], out[2][1], out[3][1])
        for k, name in enumerate(('z_lig', 'z_pocket', 'm1_lig', 'm1_pocket', 'm2_lig', 'm2_pocket')):
            assert_fp64_bound(got[k], refs[0][k], refs[1][k], f'3M s={s} {name}')
        zl, zp, hl, hp = out


ROUNDS = 2


def test_eager_conditional_rounds_against_float64():
    torch.manual_seed(5)
    ddpm = _ddpm()
    ddpm.dynamics = rec = _Recording(ddpm.dynamics)
    ligand, fixed = make_ligand([7, 5], 3)
    ligand, pocket = ddpm.normalize(ligand, make_pocket())
    lm, pm = ligand['mask'], pocket['mask']
    xh_pocket = torch.cat([pocket['x'], pocket['one_hot']], 1)
    xh_ligand = torch.cat([ligand['x'], ligand['one_hot']], 1)
    com0 = scatter_mean(pocket['x'], pm, dim=0)
    z = torch.randn(len(lm), 3 + DDPM_CFG.atom_nf)
    z[:, :3], xh_pocket[:, :3] = ddpm.remove_mean_batch(z[:, :3], xh_pocket[:, :3], lm, pm)
    hist = ddpm._empty_history(z, 'dpmpp_3m')
    t_table, coef = ddpm._fast_tables(N_STEPS, 'dpmpp_3m', 0.0, 'cpu')
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
                                          com0, fixed.view(-1, 1), lm, pm, 'dpmpp_3m', 0.0, last)
            assert len(noises) == 1 + (not last), 'draws: known part, re-noise'
            args = (z, xh_pocket, *hist, rec.out[0], noises[0], None if last else noises[1], coef[s:s + 1].expand(2, -1),
                    anc[s:s + 1, 3:].expand(2, -1), xh_ligand, com0, fixed, lm, pm, last)
            refs = [cond_round3_ref(*args, d) for d in (torch.float32, torch.float64)]
            for i, (name, got) in enumerate(zip(('z', 'pocket', 'm1', 'm2'), out[:2] + tuple(out[2]))):
                assert_fp64_bound(got, refs[0][i], refs[1][i], f'3M s={s} u={u} {name}')
            z, xh_pocket, hist = out


def test_eager_joint_rounds_against_float64():
    torch.manual_seed(6)
    ddpm = _ddpm(JOINT_CFG, joint=True)
    ddpm.dynamics = rec = _Recording(ddpm.dynamics)
    ligand, fixed = make_ligand([7, 5], 2)
    ligand, pocket = ddpm.normalize(ligand, make_pocket())
    lm, pm = ligand['mask'], pocket['mask']
    fp = torch.ones(len(pm))
    fp[::4] = 0
    xl, xp = torch.cat([ligand['x'], ligand['one_hot']], 1), torch.cat([pocket['x'], pocket['one_hot']], 1)
    zl, zp = ddpm.sample_combined_position_feature_noise(lm, pm)
    hist = (ddpm._empty_history(zl, 'dpmpp_3m'), ddpm._empty_history(zp, 'dpmpp_3m'))
    t_table, coef = ddpm._fast_tables(N_STEPS, 'dpmpp_3m', 0.0, 'cpu')
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
                                                         fixed.view(-1, 1), fp.view(-1, 1), lsel, psel, lm, pm, 'dpmpp_3m', 0.0,
                                                         commit)
            if not commit:
                zl1, zp1, h1 = ddpm._joint_renoise(zl1, zp1, h1, ddpm.gamma((sa + 1) / N_STEPS), gs, lm, pm)
            assert len(noises) == 1 + (not commit), 'draws: known part, jump back'
            (m1l, m2l), (m1p, m2p) = hist
            args = (zl, zp, m1l, m1p, m2l, m2p, *rec.out, as_kernel(noises[0]), None if commit else as_kernel(noises[1]),
                    coef[s:s + 1].expand(2, -1), anc[s:s + 1, 3:].expand(2, -1), xl, xp, fixed, fp, lm, pm, commit)
            refs = [joint_round3_ref(*args, d) for d in (torch.float32, torch.float64)]
            got = (zl1, zp1, h1[0][0], h1[1][0], h1[0][1], h1[1][1])
            for i, name in enumerate(('z_lig', 'z_pocket', 'm1_lig', 'm1_pocket', 'm2_lig', 'm2_pocket')):
                assert_fp64_bound(got[i], refs[0][i], refs[1][i], f'3M s={s} u={u} {name}')
            zl, zp, hist = zl1, zp1, h1


# ---- 3. convergence order ----------------------------------------------------------------------------------------------
T_ORDER = 3200
N_ORDER = (50, 100, 200, 400, 800)


def _solve(ddpm, den, z, pocket, lm, pm, N, sampler):
    """The sampler's formulas in float64 (fast_coefficients, the cases modules) from z_T down to z_0."""
    from fast_sampler_cases import multistep_ref
    gs, gt = _gammas(ddpm, N)
    coef = fast_coefficients(gs, gt, sampler, 0.0)
    t_all = ((torch.arange(N) + 1) / N).double()
    m1, m2 = torch.zeros_like(z), torch.zeros_like(z)
    for s in reversed(range(N)):
        c = coef[s:s + 1].expand(int(lm.max()) + 1, -1)
        eps = den(z, pocket, t_all[s].expand(c.shape[0], 1), lm, pm)
        if sampler == 'dpmpp_2m':
            z, pocket, m1 = multistep_ref(z, eps, m1, c, pocket, lm, pm, torch.float64)
        else:
            z, pocket, m1, m2 = multistep3_ref(z, eps, m1, m2, c, pocket, lm, pm, torch.float64)
    return z


@pytest.mark.timeout(1800)
def test_convergence_order():
    cfg = DDPM_CFG.with_(edge_cutoff_pocket=None, edge_cutoff_interaction=None)     # continuous field (DESIGN §5)
    sd = syn.synthetic_state_dict(cfg, 11)
    ddpm = _ddpm(cfg, T=T_ORDER)

    def den(z, pocket, t, lm, pm):
        return egnn_oracle.denoiser_forward(cfg, sd, z, pocket, t, lm, pm, dtype=torch.float64)[0]

    g = torch.Generator().manual_seed(5)
    n_lig, n_poc = [5, 4], [8, 6]
    lm, pm = torch.repeat_interleave(torch.arange(2), torch.tensor(n_lig)), torch.repeat_interleave(torch.arange(2), torch.tensor(n_poc))
    z = torch.randn((sum(n_lig), 3 + cfg.atom_nf), generator=g, dtype=torch.float64)
    pocket = torch.cat([torch.randn((sum(n_poc), 3), generator=g, dtype=torch.float64) * 1.5,
                        torch.nn.functional.one_hot(torch.arange(sum(n_poc)) % cfg.residue_nf, cfg.residue_nf).double() / 4], 1)
    z[:, :3], pocket[:, :3] = ddpm.remove_mean_batch(z[:, :3], pocket[:, :3], lm, pm)
    ref = _solve(ddpm, den, z, pocket, lm, pm, T_ORDER, 'dpmpp_3m')
    err, orders = {}, {}
    for sampler in ('dpmpp_2m', 'dpmpp_3m'):
        err[sampler] = [float((_solve(ddpm, den, z, pocket, lm, pm, N, sampler) - ref).abs().max()) for N in N_ORDER]
        orders[sampler] = [math.log2(a / b) for a, b in zip(err[sampler], err[sampler][1:])]
        print(sampler, ['%.3e' % e for e in err[sampler]], ['%.3f' % o for o in orders[sampler]])
    for N, e2, e3 in zip(N_ORDER, err['dpmpp_2m'], err['dpmpp_3m']):
        if N >= 100:
            assert e3 < e2, f'N={N}: 3M error {e3:.3e} not below 2M error {e2:.3e}'
    # measured 1.99, 2.73, 2.66, 2.36: above 2M's order, below 3 at these N (DESIGN §15: the first-order first step)
    assert min(orders['dpmpp_3m'][-2:]) >= 2.25, f"DPM-Solver++(3M) observed order {orders['dpmpp_3m']}"
    assert orders['dpmpp_2m'][-1] >= 1.7, f"DPM-Solver++(2M) observed order {orders['dpmpp_2m']}"


# ---- 4. refusals before any draw ---------------------------------------------------------------------------------------
def _refused(call, match=None):
    state = torch.random.get_rng_state()
    with pytest.raises(ValueError, match=match):
        call()
    assert torch.equal(state, torch.random.get_rng_state()), 'a draw happened before the arguments were refused'


def _copy(d):
    return {k: v.clone() for k, v in d.items()}


def test_3m_is_a_sampler():
    check_sampler('dpmpp_3m', 0.0)
    for eta in (0.5, 1.0, -0.1):
        with pytest.raises(ValueError):
            check_sampler('dpmpp_3m', eta)


def test_refusals_before_any_draw():
    cond, joint, simple = _ddpm(), _ddpm(JOINT_CFG, joint=True), _ddpm(cls=SimpleConditionalDDPM)
    ligand, fixed = make_ligand([7, 5], 3)
    pocket = make_pocket()
    pf = torch.ones(len(pocket['mask']))
    n_lig = torch.tensor([5, 6])
    # eta must be 0, at every entry point
    _refused(lambda: cond.sample_given_pocket(_copy(pocket), n_lig, sampler='dpmpp_3m', eta=0.5))
    _refused(lambda: joint.sample(2, n_lig, torch.tensor([7, 8]), sampler='dpmpp_3m', eta=0.5))
    _refused(lambda: sample_given_pocket_sharded(cond, _copy(pocket), n_lig, sampler='dpmpp_3m', eta=0.5))
    _refused(lambda: cond.inpaint(_copy(ligand), _copy(pocket), fixed, sampler='dpmpp_3m', eta=0.5))
    _refused(lambda: cond.diversify(_copy(ligand), _copy(pocket), 5, sampler='dpmpp_3m', eta=0.5))
    _refused(lambda: joint.inpaint(_copy(ligand), _copy(pocket), fixed, pf, sampler='dpmpp_3m', eta=0.5))
    # the joint inpaint with jumps over several steps, SimpleConditionalDDPM's RePaint paths, diversify's grid
    _refused(lambda: joint.inpaint(_copy(ligand), _copy(pocket), fixed, pf, resamplings=2, jump_length=2, sampler='dpmpp_3m'),
             match='jump_length')
    _refused(lambda: simple.inpaint(_copy(ligand), _copy(pocket), fixed, sampler='dpmpp_3m'))
    _refused(lambda: simple.diversify(_copy(ligand), _copy(pocket), 5, sampler='dpmpp_3m'))
    _refused(lambda: cond.diversify(_copy(ligand), _copy(pocket), 5, sampler='dpmpp_3m', denoising_steps=6))


def _lightning(mode):
    from argparse import Namespace
    from diffsbdd_b200.lightning_modules import LigandPocketDDPM
    egnn = Namespace(device='cpu', joint_nf=16, hidden_nf=64, n_layers=2, attention=True, tanh=True, norm_constant=1,
                     inv_sublayers=1, sin_embedding=False, normalization_factor=100, aggregation_method='sum',
                     edge_cutoff_ligand=None, edge_cutoff_pocket=5.0, edge_cutoff_interaction=5.0,
                     reflection_equivariant=False)
    diff = Namespace(diffusion_steps=20, diffusion_noise_schedule='polynomial_2', diffusion_noise_precision=5e-4,
                     diffusion_loss_type='l2', normalize_factors=[1, 4])
    return LigandPocketDDPM(outdir=None, dataset='crossdock', datadir=None, batch_size=4, lr=1e-3, egnn_params=egnn,
                            diffusion_params=diff, num_workers=0, augment_noise=0, augment_rotation=False, clip_grad=True,
                            eval_epochs=1, eval_params=Namespace(), visualize_sample_epoch=1, visualize_chain_epoch=1,
                            auxiliary_loss=False, loss_params=Namespace(), mode=mode,
                            node_histogram=[[1.0, 2.0], [3.0, 1.0]], pocket_representation='full-atom')


def test_joint_generate_ligand_tensors_refuses_3m():
    model = _lightning('joint')
    _refused(lambda: model.generate_ligand_tensors(make_pocket(), sampler='dpmpp_3m'), match='joint model')


def test_simple_conditional_samples_with_3m():
    torch.manual_seed(7)
    out = _ddpm(cls=SimpleConditionalDDPM).sample_given_pocket(make_pocket(), torch.tensor([5, 6]), timesteps=5,
                                                               sampler='dpmpp_3m')
    assert bool(torch.isfinite(out[0]).all())
