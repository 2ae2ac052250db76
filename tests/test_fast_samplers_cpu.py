"""CPU: the few-step samplers 'ddim' and 'dpmpp_2m' (DESIGN §13) against float64, without a GPU.

* coefficient tables: DDIM at eta = 1 is the ancestral step of ``_schedule_tables`` / ``_joint_tables`` (float64 to 1e-12;
  fp32 within half an ulp of float64, and from the fp32 ancestral tables by no more than their own fp32 rounding) for the
  polynomial, cosine and learned schedules; the first 2M step is DDIM at eta = 0;
* the eager engine, teacher-forced: each fp32 step against the float64 restatement of its formulas on the same inputs;
* convergence order on a cut-off-free model with the float64 oracle denoiser: DDIM is first order, 2M second order;
* argument validation before any draw, including the refusal of the joint model's inpainting route.
"""
import math
from argparse import Namespace

import pytest
import torch

from ddpm_cases import DDPM_CFG, HIST, JOINT_CFG, assert_fp64_bound, make_pocket
from fast_sampler_cases import ddim_ref, joint_ddim_ref, joint_multistep_ref, multistep_ref
from diffsbdd_b200 import synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM
from diffsbdd_b200.distributed import sample_given_pocket_sharded
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion, check_sampler, fast_coefficients, num_nodes_to_batch_mask
from oracle import egnn_oracle
from oracle.cpu_denoiser import OracleDynamics

SCHEDULES = ('polynomial_2', 'cosine', 'learned')
T_TABLE = 500


def _ddpm(cfg=DDPM_CFG, joint=False, T=20, schedule='polynomial_2', dynamics=None):
    cls = EnVariationalDiffusion if joint else ConditionalDDPM
    dyn = dynamics if dynamics is not None else OracleDynamics(cfg, syn.synthetic_state_dict(cfg, 5))
    ddpm = cls(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=T, noise_schedule=schedule,
               noise_precision=5e-4, loss_type='vlb' if schedule == 'learned' else 'l2', norm_values=(1, 4),
               size_histogram=HIST)
    return ddpm.eval()


def _gammas(ddpm, N):
    s_int = torch.arange(N).view(-1, 1)
    return ddpm.gamma(s_int / N).detach(), ddpm.gamma((s_int + 1) / N).detach()


# ---- 1. coefficient tables ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('schedule', SCHEDULES)
@pytest.mark.parametrize('N', [T_TABLE, T_TABLE // 5, T_TABLE // 50])
def test_ddim_eta1_is_the_ancestral_step(schedule, N):
    torch.manual_seed(0)
    ddpm = _ddpm(T=T_TABLE, schedule=schedule)
    gs, gt = _gammas(ddpm, N)
    # float64: the ancestral coefficients of the reference's ops evaluated on the same (fp32) gammas in float64
    g64s, g64t = gs.double(), gt.double()
    sigma2_ts, sigma_ts, alpha_ts = ddpm.sigma_and_alpha_t_given_s(g64t, g64s, g64s)
    sigma_s, sigma_t = ddpm.sigma(g64s, g64s), ddpm.sigma(g64t, g64s)
    anc = torch.cat([alpha_ts, sigma2_ts / alpha_ts / sigma_t, sigma_ts * sigma_s / sigma_t], dim=1)
    got = fast_coefficients(gs, gt, 'ddim', 1.0)
    assert got.dtype == torch.float64
    rel = ((got - anc).abs() / anc.abs()).max()
    assert rel <= 1e-12, f'{schedule} N={N}: DDIM(eta=1) table vs ancestral, relative {rel:.3e}'
    # fp32: the DDIM table is the float64 ancestral coefficient correctly rounded (half an ulp).  The ancestral fp32 tables
    # carry the rounding of their fp32 ops (the softplus difference of sigma^2_{t|s} cancels: hundreds of ulp at N = T), so
    # they may differ from it by that error and half an ulp more, no further.
    _, fast = ddpm._fast_tables(N, 'ddim', 1.0, 'cpu')
    _, cond = ddpm._schedule_tables(N, N, 'cpu')
    _, joint = EnVariationalDiffusion._joint_tables(ddpm, N, 1, 'cpu')
    ulp = torch.exp2(torch.floor(torch.log2(anc.abs())) - 23)
    assert float(((fast.double() - anc).abs() / ulp).max()) <= 0.5 + 1e-6, f'{schedule} N={N}: fp32 table not rounded'
    for name, ref in (('_schedule_tables', cond[:, :3]), ('_joint_tables', joint[:, :3])):
        own = (ref.double() - anc).abs() / ulp
        gap = (fast.double() - ref.double()).abs() / ulp
        assert bool((gap <= own + 0.5 + 1e-6).all()), f'{schedule} N={N}: fp32 DDIM(eta=1) table vs {name}'


@pytest.mark.parametrize('schedule', SCHEDULES)
def test_first_2m_step_is_ddim_eta0(schedule):
    torch.manual_seed(0)
    ddpm = _ddpm(T=T_TABLE, schedule=schedule)
    gs, gt = _gammas(ddpm, T_TABLE // 5)
    ddim, m2 = fast_coefficients(gs, gt, 'ddim', 0.0)[-1], fast_coefficients(gs, gt, 'dpmpp_2m')[-1]
    assert m2[4] == 0 and (fast_coefficients(gs, gt, 'dpmpp_2m')[:-1, 4] > 0).all()
    z, eps = torch.randn(50, dtype=torch.float64), torch.randn(50, dtype=torch.float64)
    a = z / ddim[0] - ddim[1] * eps
    b = m2[0] * z + m2[1] * ((z - m2[3] * eps) * m2[2])
    assert float((a - b).abs().max()) <= 1e-12 * float(a.abs().max())
    assert ddim[2] == 0


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


RUNS = [('ddim', 0.0), ('ddim', 0.5), ('dpmpp_2m', 0.0)]
N_STEPS = 10


@pytest.mark.parametrize('sampler,eta', RUNS)
def test_eager_conditional_steps_against_float64(sampler, eta):
    torch.manual_seed(3)
    ddpm = _ddpm()
    ddpm.dynamics = rec = _Recording(ddpm.dynamics)
    pocket = make_pocket()
    _, pocket = ddpm.normalize(pocket=pocket)
    n_lig = [7, 5]
    lm, pm = num_nodes_to_batch_mask(2, torch.tensor(n_lig), 'cpu'), pocket['mask']
    xh_pocket = torch.cat([pocket['x'], pocket['one_hot']], 1)
    z = torch.randn(sum(n_lig), 3 + DDPM_CFG.atom_nf)
    z[:, :3], xh_pocket[:, :3] = ddpm.remove_mean_batch(z[:, :3], xh_pocket[:, :3], lm, pm)
    hist = ddpm._empty_history(z, sampler)
    t_table, coef = ddpm._fast_tables(N_STEPS, sampler, eta, 'cpu')
    noises = []
    lig_noise = ddpm._lig_noise
    ddpm._lig_noise = lambda *a: noises.append(lig_noise(*a)) or noises[-1]
    for s in reversed(range(N_STEPS)):
        noises.clear()
        c = coef[s:s + 1].expand(2, -1)
        z1, p1, h1 = ddpm._fast_step(s, t_table[s].expand(2, 1), coef[s:s + 1], z, xh_pocket, hist, lm, pm, sampler, eta)
        eps = rec.out[0]
        assert len(noises) == (1 if eta > 0 else 0)
        if sampler == 'ddim':
            refs = [ddim_ref(z, eps, noises[0] if noises else None, c, xh_pocket, lm, pm, d) for d in (torch.float32, torch.float64)]
        else:
            refs = [multistep_ref(z, eps, *hist, c, xh_pocket, lm, pm, d) for d in (torch.float32, torch.float64)]
        got = (z1, p1) + h1
        for k, name in enumerate(('z', 'pocket', 'hist')[:len(got)]):
            assert_fp64_bound(got[k], refs[0][k], refs[1][k], f'{sampler} eta={eta} s={s} {name}')
        z, xh_pocket, hist = z1, p1, h1


@pytest.mark.parametrize('sampler,eta', RUNS)
def test_eager_joint_steps_against_float64(sampler, eta):
    torch.manual_seed(4)
    ddpm = _ddpm(JOINT_CFG, joint=True)
    ddpm.dynamics = rec = _Recording(ddpm.dynamics)
    n_lig, n_poc = [6, 4], [9, 12]
    lm, pm = num_nodes_to_batch_mask(2, torch.tensor(n_lig), 'cpu'), num_nodes_to_batch_mask(2, torch.tensor(n_poc), 'cpu')
    zl, zp = ddpm.sample_combined_position_feature_noise(lm, pm)
    hl, hp = ddpm._empty_history(zl, sampler), ddpm._empty_history(zp, sampler)
    t_table, coef = ddpm._fast_tables(N_STEPS, sampler, eta, 'cpu')
    noises = []
    draw = ddpm.sample_combined_position_feature_noise
    ddpm.sample_combined_position_feature_noise = lambda *a: noises.append(draw(*a)) or noises[-1]
    for s in reversed(range(N_STEPS)):
        noises.clear()
        c = coef[s:s + 1].expand(2, -1)
        out = ddpm._joint_fast_step(s, t_table[s].expand(2, 1), coef[s:s + 1], zl, zp, hl, hp, lm, pm, sampler, eta)
        eps_l, eps_p = rec.out
        assert len(noises) == (1 if eta > 0 else 0)
        if sampler == 'ddim':
            nz = None
            if noises:
                el, ep = noises[0]
                nz = (torch.cat((el[:, :3], ep[:, :3])), el[:, 3:], ep[:, 3:])
            refs = [joint_ddim_ref(zl, zp, eps_l, eps_p, nz, c, lm, pm, d) for d in (torch.float32, torch.float64)]
        else:
            refs = [joint_multistep_ref(zl, zp, eps_l, eps_p, *hl, *hp, c, lm, pm, d) for d in (torch.float32, torch.float64)]
        got = out[:2] + out[2] + out[3]
        assert len(got) == len(refs[0])
        for k, name in enumerate(('z_lig', 'z_pocket', 'hist_lig', 'hist_pocket')[:len(refs[0])]):
            assert_fp64_bound(got[k], refs[0][k], refs[1][k], f'{sampler} eta={eta} s={s} {name}')
        zl, zp, hl, hp = out


# ---- 3. convergence order ----------------------------------------------------------------------------------------------
T_ORDER = 3200
N_ORDER = (50, 100, 200, 400, 800)


def _solve(ddpm, den, z, pocket, lm, pm, N, sampler):
    """The sampler's formulas in float64 (fast_coefficients, fast_sampler_cases) from z_T down to z_0."""
    gs, gt = _gammas(ddpm, N)
    coef = fast_coefficients(gs, gt, sampler, 0.0)
    t_all = ((torch.arange(N) + 1) / N).double()
    hist = torch.zeros_like(z)
    for s in reversed(range(N)):
        c = coef[s:s + 1].expand(int(lm.max()) + 1, -1)
        eps = den(z, pocket, t_all[s].expand(c.shape[0], 1), lm, pm)
        if sampler == 'ddim':
            z, pocket = ddim_ref(z, eps, None, c, pocket, lm, pm, torch.float64)
        else:
            z, pocket, hist = multistep_ref(z, eps, hist, c, pocket, lm, pm, torch.float64)
    return z


@pytest.mark.timeout(900)
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
    ref = _solve(ddpm, den, z, pocket, lm, pm, T_ORDER, 'dpmpp_2m')
    orders = {}
    for sampler in ('ddim', 'dpmpp_2m'):
        err = [float((_solve(ddpm, den, z, pocket, lm, pm, N, sampler) - ref).abs().max()) for N in N_ORDER]
        orders[sampler] = [math.log2(a / b) for a, b in zip(err, err[1:])]
        print(sampler, ['%.3e' % e for e in err], ['%.3f' % o for o in orders[sampler]])
    assert 0.8 <= orders['ddim'][-1] <= 1.2, f"DDIM observed order {orders['ddim']}"
    assert orders['dpmpp_2m'][-1] >= 1.7, f"DPM-Solver++(2M) observed order {orders['dpmpp_2m']}"


# ---- 4. argument validation --------------------------------------------------------------------------------------------
BAD = [('euler', 0.0), ('ddim', -0.1), ('ddim', 1.5), ('ddim', float('nan')), ('dpmpp_2m', 0.3), ('ddpm', 0.5)]


@pytest.mark.parametrize('sampler,eta', BAD)
def test_invalid_sampler_arguments_raise_before_any_draw(sampler, eta):
    with pytest.raises(ValueError):
        check_sampler(sampler, eta)
    cond, joint = _ddpm(), _ddpm(JOINT_CFG, joint=True)
    state = torch.random.get_rng_state()
    with pytest.raises(ValueError):
        cond.sample_given_pocket(make_pocket(), torch.tensor([5, 6]), sampler=sampler, eta=eta)
    with pytest.raises(ValueError):
        joint.sample(2, torch.tensor([5, 6]), torch.tensor([7, 8]), sampler=sampler, eta=eta)
    with pytest.raises(ValueError):
        sample_given_pocket_sharded(cond, make_pocket(), torch.tensor([5, 6]), sampler=sampler, eta=eta)
    assert torch.equal(state, torch.random.get_rng_state()), 'a draw happened before the arguments were refused'


@pytest.mark.parametrize('sampler,eta', [('ddpm', 0.0), ('ddim', 0.0), ('ddim', 1.0), ('dpmpp_2m', 0.0)])
def test_valid_sampler_arguments(sampler, eta):
    check_sampler(sampler, eta)


def _lightning(mode):
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


@pytest.mark.parametrize('sampler,eta', [('ddim', 0.0), ('ddim', 0.5), ('dpmpp_2m', 0.0)])
def test_joint_generate_ligand_tensors_refuses_fast_samplers(sampler, eta):
    model = _lightning('joint')
    pocket = make_pocket(next(model.parameters()).device)
    state = torch.random.get_rng_state()
    with pytest.raises(ValueError, match='joint model'):
        model.generate_ligand_tensors(pocket, sampler=sampler, eta=eta)
    assert torch.equal(state, torch.random.get_rng_state())
    with pytest.raises(ValueError):
        _lightning('pocket_conditioning').generate_ligand_tensors(pocket, sampler='dpmpp_2m', eta=0.5)


def test_sharded_sampling_forwards_the_sampler():
    calls = []

    class _Recorder:
        n_dims, atom_nf, residue_nf = 3, DDPM_CFG.atom_nf, DDPM_CFG.residue_nf

        def sample_given_pocket(self, pocket, n_lig, timesteps=None, **kw):
            calls.append(kw)
            nl = int(n_lig.sum())
            return (torch.zeros((nl, 3 + self.atom_nf)), torch.zeros((len(pocket['mask']), 3 + self.residue_nf)),
                    torch.zeros(nl, dtype=torch.int64), pocket['mask'])

    sample_given_pocket_sharded(_Recorder(), make_pocket(), torch.tensor([5, 6]), sampler='ddim', eta=0.25)
    sample_given_pocket_sharded(_Recorder(), make_pocket(), torch.tensor([5, 6]))
    assert calls == [{'sampler': 'ddim', 'eta': 0.25}, {}]
