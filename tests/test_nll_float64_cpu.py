"""CPU: pins the float64 restatement of the likelihood evaluation (tests/nll_float64_cases.py) itself, so that a failure of
the GPU comparison (tests/test_gpu_nll_float64.py) points at the kernels.

The restatement is held, in float32 and fed the eager engine's own noise and denoiser outputs, to the eager ``forward`` of
every NLL case (every entry of the return tuple and of ``info``); in float64 to the goldens of the unmodified reference,
among them two at the production schedule (T = 500) whose injected timestep draw holds t = 1 and t = T; its
``log p(h | z_0)`` to an independent evaluation with scipy's normal CDF; the schedule to the module's fp32 table; and the
``LigandPocketDDPM.forward`` assembly (loss_t, loss_0, nll, info means) with and without virtual nodes.  The reference's
own ``LigandPocketDDPM`` needs pytorch_lightning to import, which is not installed, so the facade has no golden: the hand
restatement from lightning_modules.py:236-302 is its only check."""
import os
from argparse import Namespace

import numpy as np
import pytest
import torch
from scipy.special import log_ndtr, logsumexp, ndtr

import nll_float64_cases as nc
from ddpm_cases import DDPM_CFG, JOINT_CFG, OracleDynamics, make_pocket
from nll_cases import NLL_CASES, NLL_HIST, RETURN_NAMES, ddpm_kwargs, make_case_ligand
from diffsbdd_b200 import synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM, SimpleConditionalDDPM
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion, PredefinedNoiseSchedule
from diffsbdd_b200.lightning_modules import LigandPocketDDPM

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'nll')
CLASSES = {'conditional': ConditionalDDPM, 'simple': SimpleConditionalDDPM, 'joint': EnVariationalDiffusion}
ALL_CASES = {**NLL_CASES, **nc.NLL_T500_CASES}


def _case(name):
    """(spec, ddpm on the eager engine with the oracle denoiser, ligand, pocket, injected timestep draw or None)."""
    spec = ALL_CASES[name]
    gold = np.load(os.path.join(GOLD, name + '.npz'))
    cfg, wseed = (JOINT_CFG, 6) if spec['model'] == 'joint' else (DDPM_CFG, 5)
    ddpm = CLASSES[spec['model']](dynamics=OracleDynamics(cfg, syn.synthetic_state_dict(cfg, wseed)), **ddpm_kwargs(spec))
    ddpm.gamma.load_state_dict({k[len('gamma.'):]: torch.from_numpy(gold[k]) for k in gold.files if k.startswith('gamma.')})
    ddpm.loop_engine = 'eager'
    if name in nc.NLL_T500_CASES:
        pocket = syn.synthetic_pocket(DDPM_CFG, nc.T500_POCKET, seed=31, spread=3.0)
        t_inject = torch.tensor(nc.T500_STEPS)
    else:
        pocket, t_inject = make_pocket(), None
    return spec, ddpm.eval(), make_case_ligand(spec), pocket, t_inject, gold


def _run_recorded(name):
    spec, ddpm, ligand, pocket, t_inject, gold = _case(name)
    raw = ({k: v.clone() for k, v in ligand.items()}, {k: v.clone() for k, v in pocket.items()})
    torch.manual_seed(spec['seed'])
    with nc.ForwardRecorder(ddpm, t_inject) as rec:
        out = ddpm(ligand, pocket, return_info=True)
    return spec, ddpm, raw, rec, out, gold


def _assert_matches(r, out, rtol, atol, what):
    for key, got in zip(RETURN_NAMES, out[:-1]):
        want = r.out[key]
        assert tuple(got.shape) == tuple(want.shape), (what, key)
        assert torch.allclose(got.double(), want.double(), rtol=rtol, atol=atol), (what, key, got, want)
    assert sorted(out[-1]) == sorted(r.info), what
    for k, v in out[-1].items():
        assert torch.allclose(v.double(), r.info[k].double(), rtol=rtol, atol=atol), (what, k, v, r.info[k])


@pytest.mark.parametrize('name', sorted(ALL_CASES))
def test_restatement_reproduces_eager_forward_and_reference_golden(name):
    spec, ddpm, (ligand, pocket), rec, out, gold = _run_recorded(name)
    kind = spec['model']
    eps_t, eps_0 = rec.eps(kind)
    # float32, fed the eager engine's noise and denoiser outputs: the eager forward to fp32 rounding
    r32 = nc.restate_forward(kind, ddpm, NLL_HIST, ligand, pocket, out[10], eps_t, eps_0, rec.nets(), torch.float32)
    _assert_matches(r32, out, rtol=2e-5, atol=2e-5, what='float32')
    for call, z in zip(rec.dyn, (r32.z_t, r32.z_0)):           # and the denoiser saw the z the restatement builds
        assert torch.allclose(call[0][0], z[0], rtol=1e-5, atol=1e-5)
        assert torch.allclose(call[0][1], z[1], rtol=1e-5, atol=1e-5)
    # float64 against what the unmodified reference returned, at the goldens' tolerance
    r64 = nc.restate_forward(kind, ddpm, NLL_HIST, ligand, pocket, out[10], eps_t, eps_0, rec.nets(), torch.float64)
    # (a learned schedule evaluated in fp32 carries 3 to 4 digits of gamma: its 1024-wide layer is summed in fp32 and gamma
    # is a ratio of differences of such sums, so the reference's own SNR_weight is 4e-4 and xh_lig_hat 1e-4 from float64)
    for key in RETURN_NAMES:
        want = torch.from_numpy(gold[key]).double()
        rtol = 1e-3 if spec['schedule'] == 'learned' else 1e-5
        assert torch.allclose(r64.out[key].double(), want, rtol=rtol, atol=1e-5), (key, r64.out[key], want)
    for k, v in r64.info.items():
        assert torch.allclose(v, torch.from_numpy(gold['info_' + k]).double(), rtol=1e-5, atol=1e-5), k


@pytest.mark.parametrize('name', sorted(nc.NLL_T500_CASES))
def test_forward_matches_reference_golden_at_both_ends_of_the_production_schedule(name):
    """As test_nll_cpu.test_forward_matches_reference_golden, with the timestep draw injected: t = 1, T, 137, 420."""
    spec, ddpm, _, rec, out, gold = _run_recorded(name)
    assert out[10].tolist() == [float(t) for t in nc.T500_STEPS]
    for key, got in zip(RETURN_NAMES, out[:-1]):
        want = torch.from_numpy(gold[key])
        assert tuple(got.shape) == tuple(want.shape), key
        assert torch.allclose(got.float(), want.float(), atol=1e-5, rtol=1e-5), (key, got, want)
    assert sorted('info_' + k for k in out[-1]) == sorted(k for k in gold.files if k.startswith('info_'))
    for k, v in out[-1].items():
        assert torch.allclose(v, torch.from_numpy(gold['info_' + k]), atol=1e-5, rtol=1e-5), k


def test_log_ph_against_scipy_normal_cdf():
    """log p(h | z_0) of one node on a grid of (offset of the true class from its centre, s0), away from the 1e-10 floor's
    reach (the floor is part of the operation; scipy's tails have none): every class probability is at least 1e-4."""
    K, nv, nb = 5, 4.0, 0.0
    rows, want = [], []
    for s0 in (0.3, 0.5, 1.0, 2.0, 10.0):
        for off in np.linspace(-1.5, 1.5, 13):
            for k in (0, 2, 4):
                un = np.zeros(K)                                  # un-normalised z_0.h: 1 + off at class k, else noise-free 0
                un[k] = 1 + off
                ctr = un - 1
                # independent: log of a CDF difference from log_ndtr, log-sum-exp by scipy
                lp = np.array([np.log(ndtr((c + 0.5) / s0) - ndtr((c - 0.5) / s0)) if abs(c) < 3 * s0 else
                               log_ndtr(-(abs(c) - 0.5) / s0) + np.log1p(-np.exp(log_ndtr(-(abs(c) + 0.5) / s0)
                                                                                 - log_ndtr(-(abs(c) - 0.5) / s0)))
                               for c in ctr])
                if lp.min() < np.log(1e-4):
                    continue
                rows.append((un / nv, np.eye(K)[k] / nv, s0))
                want.append(lp[k] - logsumexp(lp))
    assert len(rows) > 100
    z = torch.tensor(np.array([r[0] for r in rows]))
    oh = torch.tensor(np.array([r[1] for r in rows]))
    s0 = torch.tensor([r[2] for r in rows])
    node, _, _ = nc.log_ph_nodes(z, oh, s0, nv, nb, torch.float64)
    assert np.allclose(node.numpy(), want, rtol=0, atol=2e-6)     # 1e-10 / 1e-4 = 1e-6 is the floor's own contribution
    node32, _, slack = nc.log_ph_nodes(z.float(), oh.float(), s0.float(), nv, nb, torch.float32)
    assert float((node32.double() - node).abs().max()) < 1e-4


def test_all_classes_floored_gives_minus_log_k():
    z = torch.full((3, 7), 9.0, dtype=torch.float64)            # every class centre 35 widths away
    oh = torch.eye(7, dtype=torch.float64)[:3] / 4.0
    for dtype in (torch.float64, torch.float32):
        node, _, slack = nc.log_ph_nodes(z, oh, torch.ones(3), 4.0, 0.0, dtype)
        assert torch.allclose(node.double(), torch.full((3,), -np.log(7.0), dtype=torch.float64), atol=1e-6)
    assert float(slack.max()) == 0.0


def test_polynomial_2_schedule_table_against_float64():
    """gamma, alpha, sigma and SNR_weight at every t of the production schedule (T = 500, precision 5e-4): the float64
    formula against the module's fp32 table.  gamma is stored to fp32 rounding (|gamma| < 8: at most 4.8e-7, 2.4e-7 found).
    sigma_0 = alpha_T = 0.02236 (s0 = 4 sigma_0 = 0.0894).  SNR_weight = 1 - exp(gamma_s - gamma_t) is a difference of two
    table entries: at t = 1 the step gamma_1 - gamma_0 is 1.59e-2 and the table carries 4 to 5 digits of it (relative error
    1.5e-5, the largest of all t); at t = T the step is 3.1e-2 and the relative error 1.9e-6."""
    T = 500
    g64 = nc.polynomial_gamma64(T, 5e-4)
    table = PredefinedNoiseSchedule('polynomial_2', T, 5e-4).gamma.detach()
    assert table.dtype == torch.float32 and table.shape == (T + 1,)
    g32 = table.double().numpy()
    assert np.abs(g32 - g64).max() <= 2.0 ** -24 * 8            # half an ulp below 8
    assert np.all(np.diff(g64) > 0)
    sig = lambda g: 1 / (1 + np.exp(-g))
    for f in (lambda g: np.sqrt(sig(-g)), lambda g: np.sqrt(sig(g))):
        assert np.abs(f(g32) - f(g64)).max() < 3e-7
    assert abs(np.sqrt(sig(g64[0])) - 0.02236) < 1e-5
    assert abs(np.sqrt(sig(-g64[T])) - 0.02236) < 1e-5          # alpha_T: the schedule is symmetric about precision
    snr = lambda g: 1 - np.exp(g[1:] - g[:-1])
    rel = np.abs(snr(g32) - snr(g64)) / np.abs(snr(g64))
    assert 1e-6 < rel[0] < 3e-5 and rel.max() == rel[0], rel[0]  # t = 1: 4 to 5 digits
    assert rel[T - 1] < 4e-6, rel[T - 1]                        # t = T
    assert abs((g64[1] - g64[0]) - 1.59e-2) < 1e-4 and abs((g64[T] - g64[T - 1]) - 3.14e-2) < 1e-4
    # the module's own alpha / sigma (fp32 ops on the fp32 table) against float64 on the same table
    t = torch.arange(T + 1)
    for mine, ops in ((nc.alpha_of, lambda g: torch.sqrt(torch.sigmoid(-g))), (nc.sigma_of, lambda g: torch.sqrt(torch.sigmoid(g)))):
        assert float((ops(table).double() - mine(table.double()[t])).abs().max()) < 2e-7


def _facade_model(virtual_nodes):
    cfg = DDPM_CFG
    egnn = Namespace(device='cpu', **{k: v for k, v in cfg.kwargs().items()
                                      if k not in ('atom_nf', 'residue_nf', 'n_dims', 'condition_time', 'mode',
                                                   'update_pocket_coords')})
    diff = Namespace(diffusion_steps=500, diffusion_noise_schedule='polynomial_2', diffusion_noise_precision=5.0e-4,
                     diffusion_loss_type='l2', normalize_factors=[1, 4])
    model = LigandPocketDDPM(outdir=None, dataset='crossdock', datadir=None, batch_size=3, lr=1e-3, egnn_params=egnn,
                             diffusion_params=diff, num_workers=0, augment_noise=0, augment_rotation=False, clip_grad=True,
                             eval_epochs=1, eval_params=Namespace(), visualize_sample_epoch=1, visualize_chain_epoch=1,
                             auxiliary_loss=False, loss_params=Namespace(), mode='pocket_conditioning',
                             node_histogram=NLL_HIST, pocket_representation='full-atom', virtual_nodes=virtual_nodes)
    return model


@pytest.mark.parametrize('virtual_nodes', [False, True])
def test_facade_assembly_against_float64(virtual_nodes):
    """LigandPocketDDPM.forward on the CPU (oracle denoiser, eager engine): nll per complex and every ``info`` entry against
    the float64 assembly from the run's own noise and denoiser outputs; with virtual nodes log p(N) is left out."""
    model = _facade_model(virtual_nodes)
    A = model.atom_nf
    cfg = DDPM_CFG.with_(atom_nf=A, residue_nf=model.aa_nf)
    model.ddpm.dynamics = OracleDynamics(cfg, syn.synthetic_state_dict(cfg, 5))
    model.ddpm.loop_engine = 'eager'
    model.eval()
    n_lig, n_poc = [7, 5, 9], [22, 17, 12]
    data = syn.synthetic_complex_batch(cfg, n_lig, n_poc, seed=4)
    if virtual_nodes:
        ends = np.cumsum(n_lig)
        rows = torch.cat([torch.arange(e - 2, e) for e in ends.tolist()])
        data['lig_one_hot'][rows] = 0
        data['lig_one_hot'][rows, model.virtual_atom] = 1
        data['num_virtual_atoms'] = torch.full((3,), 2)
    ligand, pocket = model.get_ligand_and_pocket(data)
    torch.manual_seed(9)
    with nc.ForwardRecorder(model.ddpm, torch.tensor([1, 500, 250])) as rec:
        nll, info = model(data)
    eps_t, eps_0 = rec.eps('conditional')
    r = nc.restate_forward('conditional', model.ddpm, NLL_HIST, ligand, pocket, torch.tensor([1, 500, 250]), eps_t, eps_0,
                           rec.nets(), torch.float64)
    want, want_info, loss_t, loss_0 = nc.facade(r.out, r.info, 500, virtual_nodes)
    assert nll.shape == (3,)
    assert torch.allclose(nll.double(), want, rtol=1e-5, atol=1e-4), (nll, want)
    assert sorted(info) == sorted(want_info)
    for k in info:
        assert torch.allclose(info[k].double(), want_info[k].double(), rtol=1e-5, atol=1e-5), (k, info[k], want_info[k])
    with_pn = want - r.out['log_pN'] if virtual_nodes else want + r.out['log_pN']
    assert float((with_pn - want).abs().min()) > 0.1             # the branch matters at this histogram
