"""GPU: likelihood evaluation (eval-mode ``forward``) on the native path — the fused per-graph loss-term kernel
(dsb_ddpm_vlb_terms) against torch ops, native forward against the eager forward and against the CPU oracle path, a full
configs[2] batch through ``LigandPocketDDPM.forward`` / ``validation_step``, and the NaN convention."""
import ctypes as C
from argparse import Namespace

import numpy as np
import pytest
import torch

from ddpm_cases import DDPM_CFG, DDPM_SHAPES, JOINT_CFG, OracleDynamics, assert_fp64_bound, ddpm_shape, make_pocket
from nll_cases import NLL_CASES, RETURN_NAMES, ddpm_kwargs, make_case_ligand
from diffsbdd_b200 import _native, synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM, SimpleConditionalDDPM
from diffsbdd_b200.config import FULLATOM_COND
from diffsbdd_b200.dynamics import EGNNDynamics
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion, scatter_add
from diffsbdd_b200.lightning_modules import LigandPocketDDPM

pytestmark = pytest.mark.gpu

CLASSES = {'conditional': ConditionalDDPM, 'simple': SimpleConditionalDDPM, 'joint': EnVariationalDiffusion}


# ---- the fused kernel against torch ops ------------------------------------------------------------------------------
def _torch_terms(side_l, side_p, lm, pm, coef, nv, nb, vnode, A, R, n):
    """The per-graph sums of dsb_ddpm_vlb_terms with the fp32 torch ops of the eager forward."""
    d = lambda x: x.float()
    xl, ztl, etl, ntl, z0l, e0l, n0l = map(d, side_l)
    coef = d(coef)
    aT, s0, at, st = (coef[:, k:k + 1] for k in range(4))
    out = torch.zeros((n, 11), device=xl.device)
    sq_t = (etl - ntl) ** 2
    sq_0 = (e0l[:, :3] - n0l[:, :3]) ** 2
    if vnode >= 0:
        virt = xl[:, 3 + vnode] != 0
        sq_t[virt, :3] = 0
        sq_0[virt] = 0

    def log_ph(z0, x, m):
        ctr = (z0[:, 3:] * nv + nb) - 1
        w = s0[m]
        cdf = lambda v: 0.5 * (1 + torch.erf(v / np.sqrt(2)))
        lp = torch.log(cdf((ctr + 0.5) / w) - cdf((ctr - 0.5) / w) + 1e-10)
        return scatter_add(((lp - torch.logsumexp(lp, 1, keepdim=True)) * (x[:, 3:] * nv + nb)).sum(1), m, dim_size=n)

    s = lambda v, m: scatter_add(v.sum(1), m, dim_size=n)
    out[:, 0], out[:, 2], out[:, 4] = s(sq_t, lm), s(sq_0, lm), log_ph(z0l, xl, lm)
    mu = aT[lm] * xl
    out[:, 5], out[:, 6] = s(mu[:, :3] ** 2, lm), s(mu[:, 3:] ** 2, lm)
    out[:, 7], out[:, 8] = s(ntl[:, :3].abs(), lm), s(ntl[:, 3:].abs(), lm)
    if side_p is not None:
        xp, etp, ntp, z0p, e0p, n0p = map(d, side_p)
        out[:, 1], out[:, 3] = s((etp - ntp) ** 2, pm), s((e0p[:, :3] - n0p[:, :3]) ** 2, pm)
        out[:, 4] += log_ph(z0p, xp, pm)
        mu = aT[pm] * xp
        out[:, 5] += s(mu[:, :3] ** 2, pm)
        out[:, 6] += s(mu[:, 3:] ** 2, pm)
        out[:, 9], out[:, 10] = s(ntp[:, :3].abs(), pm), s(ntp[:, 3:].abs(), pm)
    hat = ztl / at[lm] - ntl * st[lm] / at[lm]
    return out, hat


def _launch(side_l, side_p, lm, pm, coef, nv, nb, vnode, A, R, n):
    lib = _native.load()
    terms = torch.full((n, 11), float('nan'), device='cuda')
    hat = torch.empty_like(side_l[1])
    ptr = lambda x: None if x is None else x.data_ptr()
    _native.check(lib.dsb_ddpm_vlb_terms(*[ptr(x) for x in side_l], *[ptr(x) for x in (side_p or [None] * 6)], ptr(coef),
                                         ptr(lm), ptr(pm), len(lm), len(pm), n, A, R, nv, nb, vnode, ptr(terms), ptr(hat),
                                         C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return terms, hat


@pytest.mark.parametrize('joint,vnode', [(False, -1), (False, 4), (True, -1)])
def test_fused_vlb_terms_match_torch(joint, vnode):
    g = torch.Generator().manual_seed(11 + vnode + 10 * joint)
    n_lig, n_poc = [7, 1, 13, 150], [30, 5, 0, 180]        # ragged, a one-atom ligand, an empty pocket, > 128 rows
    A, R, n = 10, 12, 4
    nv, nb = 4.0, (0.0 if vnode >= 0 else 0.25)     # with a bias every row's normalised vnode column is non-zero
    lm = torch.repeat_interleave(torch.arange(n), torch.tensor(n_lig)).cuda()
    pm = torch.repeat_interleave(torch.arange(n), torch.tensor(n_poc)).cuda()

    def onehot_rows(rows, k):
        oh = torch.nn.functional.one_hot(torch.randint(0, k, (rows,), generator=g), k).float()
        return (oh - nb) / nv

    def side(rows, k, with_zt):
        x = torch.cat([torch.randn((rows, 3), generator=g), onehot_rows(rows, k)], 1)
        rnd = [torch.randn((rows, 3 + k), generator=g) for _ in range(6 if with_zt else 5)]
        return [t.cuda().contiguous() for t in [x] + rnd]

    side_l = side(len(lm), A, True)
    if vnode >= 0:                                # every third ligand atom virtual
        h = torch.full((A,), -nb / nv, device='cuda')
        h[vnode] = (1 - nb) / nv
        side_l[0][::3, 3:] = h
    side_p = side(len(pm), R, False) if joint else None
    coef = torch.cat([torch.rand((n, 1), generator=g) * 0.2 + 0.05, torch.rand((n, 1), generator=g) * 0.2 + 0.05,
                      torch.rand((n, 1), generator=g) * 0.8 + 0.1, torch.rand((n, 1), generator=g) * 0.8 + 0.1], 1).cuda()
    want, want_hat = _torch_terms(side_l, side_p, lm, pm, coef, nv, nb, vnode, A, R, n)
    got, hat = _launch(side_l, side_p, lm, pm, coef, nv, nb, vnode, A, R, n)
    if not joint:
        assert torch.all(got[:, [1, 3, 9, 10]] == 0)
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-5), float((got - want).abs().max())
    assert torch.allclose(hat, want_hat, rtol=1e-5, atol=1e-6)
    again, hat2 = _launch(side_l, side_p, lm, pm, coef, nv, nb, vnode, A, R, n)
    assert torch.equal(again, got) and torch.equal(hat2, hat)         # fixed-order reduction: bit for bit


@pytest.mark.parametrize('with_pocket', [False, True])
@pytest.mark.parametrize('shape', sorted(DDPM_SHAPES))
def test_fused_noise_kernel_matches_torch(shape, with_pocket):
    """dsb_ddpm_noise: z = alpha[g] xh + sigma[g] eps on ligand rows and, for the joint model, pocket rows (skipped when the
    pocket pointer is NULL), one 128-thread block per graph."""
    g = torch.Generator().manual_seed(13 + with_pocket)
    n_lig, n_poc = ddpm_shape(shape, [7, 1, 13], [30, 5, 11])
    A, R, B = 10, 12, len(n_lig)
    NL, NP = sum(n_lig), sum(n_poc)
    lm = torch.repeat_interleave(torch.arange(B), torch.tensor(n_lig)).cuda()
    pm = torch.repeat_interleave(torch.arange(B), torch.tensor(n_poc)).cuda()
    xl, el = torch.randn((NL, 3 + A), generator=g).cuda(), torch.randn((NL, 3 + A), generator=g).cuda()
    xp, ep = torch.randn((NP, 3 + R), generator=g).cuda(), torch.randn((NP, 3 + R), generator=g).cuda()
    coef = (torch.rand((B, 2), generator=g) * 0.9 + 0.05).cuda()
    zl = torch.full_like(xl, float('nan'))
    zp = torch.full_like(xp, float('nan'))
    lib = _native.load()
    ptr = lambda x: x.data_ptr() if with_pocket else None
    _native.check(lib.dsb_ddpm_noise(xl.data_ptr(), el.data_ptr(), ptr(xp), ptr(ep), coef.data_ptr(), lm.data_ptr(), pm.data_ptr(),
                                     NL, NP, B, A, R, zl.data_ptr(), ptr(zp), C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    ref = lambda x, e, m, dt: coef.to(dt)[m, 0:1] * x.to(dt) + coef.to(dt)[m, 1:2] * e.to(dt)
    assert_fp64_bound(zl, ref(xl, el, lm, torch.float32), ref(xl, el, lm, torch.float64), f'{shape} ligand')
    if with_pocket:
        assert_fp64_bound(zp, ref(xp, ep, pm, torch.float32), ref(xp, ep, pm, torch.float64), f'{shape} pocket')
    else:
        assert torch.isnan(zp).all()                 # pocket output untouched


# ---- native forward against the eager forward and the CPU oracle -------------------------------------------------------
def _build(spec, device, native, cfg=None, math_mode=None):
    cfg = cfg or (JOINT_CFG if spec['model'] == 'joint' else DDPM_CFG)
    sd = syn.synthetic_state_dict(cfg, 6 if spec['model'] == 'joint' else 5)
    if native:
        dyn = EGNNDynamics.from_config(cfg, device=device)
        dyn.load_state_dict(sd)
        if math_mode is not None:
            dyn.math_mode = math_mode
    else:
        dyn = OracleDynamics(cfg, sd, device=device)
    torch.manual_seed(0)
    kw = ddpm_kwargs(spec)
    kw.update(atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf)
    return CLASSES[spec['model']](dynamics=dyn, **kw).to(device).eval()


def _inputs(spec, device):
    lig = make_case_ligand(spec)
    return {k: v.to(device) for k, v in lig.items()}, make_pocket(device)


def _assert_outputs_close(got, want, atol, rtol):
    for key, a, b in zip(RETURN_NAMES, got[:-1], want[:-1]):
        a, b = a.detach().cpu().double(), b.detach().cpu().double()
        assert a.shape == b.shape, key
        assert torch.allclose(a, b, atol=atol, rtol=rtol), (key, float((a - b).abs().max()))
    assert sorted(got[-1]) == sorted(want[-1])
    for k in got[-1]:
        assert torch.allclose(got[-1][k].cpu().double(), want[-1][k].cpu().double(), atol=atol, rtol=rtol), k


@pytest.mark.parametrize('name', sorted(NLL_CASES))
def test_native_forward_matches_eager_forward_same_seed(name):
    spec = NLL_CASES[name]
    ddpm = _build(spec, 'cuda', native=True)
    outs = {}
    for engine in ('eager', 'auto'):
        ddpm.loop_engine = engine
        torch.manual_seed(spec['seed'])
        outs[engine] = ddpm(*_inputs(spec, 'cuda'), return_info=True)
    _assert_outputs_close(outs['auto'], outs['eager'], atol=1e-5, rtol=1e-4)


class _NoiseTape:
    """Replaces ``sample_gaussian`` so a CPU run and a GPU run consume the same noise."""

    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)

    def __call__(self, size, device):
        return torch.randn(size, generator=self.g).to(device)


@pytest.mark.parametrize('math_mode', ['3xfp16', '3xtf32', 'fp32'])
def test_native_forward_matches_cpu_oracle_with_injected_noise(math_mode, monkeypatch):
    spec = dict(NLL_CASES['cond_ragged'], n_lig=[9, 11])
    cfg = DDPM_CFG.with_(hidden_nf=128)                   # a tensor-core width
    cpu = _build(spec, 'cpu', native=False, cfg=cfg)
    cpu.loop_engine = 'eager'
    cpu.sample_gaussian = _NoiseTape(21)
    gpu = _build(spec, 'cuda', native=True, cfg=cfg, math_mode=math_mode)
    assert gpu._vlb_native('cuda')
    gpu.sample_gaussian = _NoiseTape(21)
    inp_cpu, inp_gpu = _inputs(spec, 'cpu'), _inputs(spec, 'cuda')
    # CPU and CUDA generators differ: the timestep draw is injected as well
    t_fixed = torch.tensor([[3], [17]])
    monkeypatch.setattr(torch, 'randint', lambda lo, hi, size, device=None: t_fixed.to(device))
    want = cpu(*inp_cpu, return_info=True)
    got = gpu(*inp_gpu, return_info=True)
    _assert_outputs_close(got, want, atol=1e-4, rtol=1e-4)


def test_nan_in_denoiser_output_raises():
    spec = NLL_CASES['cond_ragged']
    ddpm = _build(spec, 'cuda', native=True)
    lig, pocket = _inputs(spec, 'cuda')
    lig['x'][2, 1] = float('nan')
    with pytest.raises(ValueError, match='NaN detected in EGNN output'):
        ddpm(lig, pocket)
    torch.manual_seed(0)
    out = ddpm(*_inputs(spec, 'cuda'))                         # the sticky flag was cleared by the raise
    assert all(torch.isfinite(x).all() for x in out)


# ---- full configs[2] batch -------------------------------------------------------------------------------------------
def _full_model():
    cfg = FULLATOM_COND
    egnn = Namespace(device='cuda', **{k: v for k, v in cfg.kwargs().items()
                                       if k not in ('atom_nf', 'residue_nf', 'n_dims', 'condition_time', 'mode',
                                                    'update_pocket_coords')})
    diff = Namespace(diffusion_steps=500, diffusion_noise_schedule='polynomial_2', diffusion_noise_precision=5.0e-4,
                     diffusion_loss_type='l2', normalize_factors=[1, 4])
    model = LigandPocketDDPM(outdir=None, dataset='crossdock', datadir=None, batch_size=64, lr=1e-3, egnn_params=egnn,
                             diffusion_params=diff, num_workers=0, augment_noise=0, augment_rotation=False, clip_grad=True,
                             eval_epochs=1, eval_params=Namespace(), visualize_sample_epoch=1, visualize_chain_epoch=1,
                             auxiliary_loss=False, loss_params=Namespace(), mode='pocket_conditioning',
                             node_histogram=np.ones((27, 177)).tolist(), pocket_representation='full-atom')
    model.ddpm.dynamics.load_state_dict(syn.synthetic_state_dict(cfg, 0))
    return model.to('cuda').eval(), cfg


def test_full_config_batch_end_to_end():
    model, cfg = _full_model()
    data = syn.synthetic_complex_batch(cfg, [25] * 64, [175] * 64, seed=3)
    ligand, pocket = model.get_ligand_and_pocket(data)
    torch.manual_seed(5)
    out = model.ddpm(ligand, pocket, return_info=True)
    for key, v in zip(RETURN_NAMES, out[:-1]):
        assert torch.isfinite(v).all(), key
    nll = []
    for _ in range(2):
        torch.manual_seed(7)
        n, info = model(data)
        nll.append(n)
    assert nll[0].shape == (64,) and torch.isfinite(nll[0]).all()
    assert torch.allclose(nll[0], nll[1], rtol=2e-6, atol=0), float((nll[0] - nll[1]).abs().max())
    for k in ('error_t_lig', 'SNR_weight', 'loss_0', 'kl_prior', 'log_pN', 'eps_hat_lig_x'):
        assert torch.isfinite(info[k]), k
    res = model.validation_step(data, 0)
    assert torch.isfinite(res['loss']) and res['loss'].dim() == 0
    assert torch.isfinite(model.test_step(data, 0)['loss'])
    model.train()
    with pytest.raises(NotImplementedError):
        model(data)
