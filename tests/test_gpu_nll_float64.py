"""GPU: the likelihood evaluation (validation / test NLL) on the native path against float64.

What is fed to what.  The restatement of tests/nll_float64_cases.py (pinned on the CPU by tests/test_nll_float64_cpu.py) is
evaluated in float64 (truth) and float32 (yardstick) on exactly what each native stage received:

  a. dsb_ddpm_vlb_terms alone, inputs built as production builds them (z_0 = alpha_0 xh + sigma_0 eps, net = eps + a small
     error, one-hot h normalised by 4): configs[2], a 2000-row pocket beside a one-atom ligand, one graph, a graph id in
     neither mask, an empty pocket, an all-virtual ligand, one class, class counts 10 / 11 / 13, a non-zero bias; a
     per-node sweep of one-atom graphs over s0 in [1e-3, 10] x centre offsets (term 4 is then one node's log p(h | z_0),
     held to float64 node by node without the case-wide fp32 term of the bound); the argument checks.
  b. dsb_ddpm_noise and the conditional dsb_ddpm_ligand_update noising at t = 0 .. 500 of polynomial_2 in one launch each.
  c. the forward of each DDPM class on 500 ragged complexes, complex g at t = g + 1: centring, z_t, z_0, the eleven sums,
     xh_lig_hat, and every entry of the return tuple and of ``info`` per complex, each stage fed the native fp32 inputs
     of that stage (recorded around the stage's own method; the recorded run equals an unrecorded one bit for bit).
  d. LigandPocketDDPM.forward on the configs[2] batch (H = 256, 6 layers) in every math mode and the joint production model
     (H = 128, 5 layers): the same stages, ending at the per-complex nll and the ``info`` means.

The two denoiser calls inside c and d are not re-derived here: their outputs are taken as recorded (the denoiser has its own
float64 tests, launch by launch, in test_gpu_launches.py), so the NLL figures below are the error of everything around
the denoiser.  Bounds: R, C_EL, C_SUM, C_ERF of nll_float64_cases, the same for every case.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import nll_float64_cases as nc
import test_gpu_nll as base
from ddpm_cases import DDPM_CFG, JOINT_CFG
from nll_cases import NLL_HIST, RETURN_NAMES
from diffsbdd_b200 import _native, synthetic as syn
from diffsbdd_b200.config import FULLATOM_JOINT

pytestmark = pytest.mark.gpu

TERM_NAMES = ('error_t_lig', 'error_t_pocket', 'sq_0_x_lig', 'sq_0_x_pocket', 'log_ph', 'mu_T_x^2', 'mu_T_h^2', '|net_t.x| lig',
              '|net_t.h| lig', '|net_t.x| pocket', '|net_t.h| pocket')
S0_PRODUCTION = 4 * math.sqrt(5e-4)        # norm_value_h sigma_0 of polynomial_2 at precision 5e-4 (sigma_0^2 = precision)


def _card():
    import subprocess
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        q = torch.cuda.get_device_name(0) + ', power limit unknown'
    return q


def _ptr(x):
    return None if x is None else x.data_ptr()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _launch_terms(side_l, side_p, lm, pm, coef, nv, nb, vnode, A, R, n):
    terms = torch.full((n, 11), float('nan'), device='cuda')
    hat = torch.full_like(side_l[1], float('nan'))
    rc = _native.load().dsb_ddpm_vlb_terms(*[_ptr(x) for x in side_l], *[_ptr(x) for x in (side_p or [None] * 6)], _ptr(coef),
                                           _ptr(lm), _ptr(pm), len(lm), len(pm), n, A, R, nv, nb, vnode, _ptr(terms), _ptr(hat),
                                           _stream())
    torch.cuda.synchronize()
    return rc, terms, hat


# ---- a. the fused kernel alone -------------------------------------------------------------------------------------------
def _production_sides(lm, pm, n, A, R, nv, nb, s0, joint, g, virtual_rows=None, vnode=-1):
    """Inputs as the forward builds them.  s0 [n] = norm_value_h sigma_0 per graph."""
    sigma_0 = (s0 / nv).clamp(max=0.999)
    alpha_0 = torch.sqrt(1 - sigma_0 ** 2)
    alpha_t = torch.rand(n, generator=g) * 0.97 + 0.02
    sigma_t = torch.sqrt(1 - alpha_t ** 2)
    coef = torch.stack([torch.full((n,), 0.02236), s0, alpha_t, sigma_t], 1).float()

    def side(mask, k, lig):
        rows = len(mask)
        types = torch.randint(0, k, (rows,), generator=g)
        if lig and virtual_rows is not None:
            types[virtual_rows] = vnode
        xh = torch.cat([torch.randn((rows, 3), generator=g) * 2, (torch.nn.functional.one_hot(types, k).float() - nb) / nv], 1)
        eps_t, eps_0 = torch.randn((rows, 3 + k), generator=g), torch.randn((rows, 3 + k), generator=g)
        m = mask.cpu()
        z_t = alpha_t[m, None] * xh + sigma_t[m, None] * eps_t
        z_0 = alpha_0[m, None] * xh + sigma_0[m, None] * eps_0
        net_t = eps_t + 0.3 * torch.randn((rows, 3 + k), generator=g)
        net_0 = eps_0 + 0.3 * torch.randn((rows, 3 + k), generator=g)
        full = [xh, z_t, eps_t, net_t, z_0, eps_0, net_0]
        return [t.float().cuda().contiguous() for t in (full if lig else full[:1] + full[2:])]

    return side(lm, A, True), (side(pm, R, False) if joint else None), coef.cuda().contiguous()


def _masks(n_lig, n_poc, ids=None):
    ids = torch.arange(len(n_lig)) if ids is None else torch.tensor(ids)
    return (torch.repeat_interleave(ids, torch.tensor(n_lig)).cuda(), torch.repeat_interleave(ids, torch.tensor(n_poc)).cuda())


KERNEL_CASES = {
    # name: (ligand sizes, pocket sizes, A, R, nb, form, extra)
    'configs2_conditional': ([25] * 64, [175] * 64, 10, 10, 0.0, 'conditional', {}),
    'configs2_vnode': ([25] * 64, [175] * 64, 11, 11, 0.0, 'vnode', {}),
    'configs2_joint': ([25] * 64, [175] * 64, 10, 10, 0.0, 'joint', {}),
    'big_pocket_one_atom': ([1, 40, 3], [2000, 7, 300], 10, 20, 0.0, 'joint', {}),
    'one_graph': ([9], [31], 10, 20, 0.0, 'joint', {}),
    'absent_graph_id': ([7, 5, 6], [11, 9, 13], 10, 20, 0.0, 'joint', {'ids': [0, 1, 3], 'n': 5}),
    'empty_pocket': ([6, 8], [0, 12], 10, 20, 0.0, 'joint', {}),
    'all_virtual_ligand': ([5, 7], [9, 9], 11, 20, 0.0, 'vnode', {'all_virtual': 0}),
    'one_class': ([6, 150], [8, 3], 1, 1, 0.0, 'joint', {}),
    'classes_11_13': ([9, 130, 1], [14, 200, 6], 11, 13, 0.0, 'joint', {}),
    'bias': ([7, 12], [20, 5], 10, 13, 0.25, 'joint', {'s0': 2.0}),
    'wide_s0': ([25] * 8, [60] * 8, 10, 20, 0.0, 'joint', {'s0': 'spread'}),
}


@pytest.mark.parametrize('name', sorted(KERNEL_CASES))
def test_fused_terms_against_float64(name):
    n_lig, n_poc, A, R, nb, form, extra = KERNEL_CASES[name]
    g = torch.Generator().manual_seed(sorted(KERNEL_CASES).index(name) + 40)
    lm, pm = _masks(n_lig, n_poc, extra.get('ids'))
    n = extra.get('n', len(n_lig))
    nv = 4.0
    s0 = torch.full((n,), S0_PRODUCTION)
    if extra.get('s0') == 'spread':                 # a learned schedule can put sigma_0 anywhere: the transition region
        s0 = torch.logspace(-1, 0.5, n)
    elif 's0' in extra:
        s0 = torch.full((n,), float(extra['s0']))
    vnode, virtual_rows = -1, None
    if form == 'vnode':
        vnode = A - 1
        virtual_rows = torch.arange(0, len(lm), 3)
        if 'all_virtual' in extra:
            virtual_rows = torch.cat([virtual_rows, torch.nonzero(lm.cpu() == extra['all_virtual']).flatten()]).unique()
    side_l, side_p, coef = _production_sides(lm, pm, n, A, R, nv, nb, s0, form == 'joint', g, virtual_rows, vnode)
    rc, terms, hat = _launch_terms(side_l, side_p, lm, pm, coef, nv, nb, vnode, A, R, n)
    assert rc == 0, _native.load().dsb_last_error()
    r64 = nc.vlb_terms_ref(side_l, side_p, lm, pm, coef, nv, nb, vnode, n, torch.float64)
    r32 = nc.vlb_terms_ref(side_l, side_p, lm, pm, coef, nv, nb, vnode, n, torch.float32)
    ratios = nc.assert_sum_bound(terms, r32, r64, name, TERM_NAMES)
    hat_ratio = nc.assert_element_bound(hat, r32.hat, r64.hat, r64.hat_scale, name + ' xh_lig_hat')
    print(f'{name}: error / bound per term {[round(x, 3) for x in ratios]}, xh_lig_hat {hat_ratio:.3f}')
    if form != 'joint':
        assert torch.all(terms[:, [1, 3, 9, 10]] == 0)
    if 'ids' in extra:                              # a graph with no row in either mask: exactly zero, neighbours as without it
        absent = [i for i in range(n) if i not in extra['ids']]
        assert torch.all(terms[absent] == 0)
    if 'all_virtual' in extra:
        assert terms[extra['all_virtual'], 2] == 0 and terms[extra['all_virtual'], 7] > 0
    rc, again, hat2 = _launch_terms(side_l, side_p, lm, pm, coef, nv, nb, vnode, A, R, n)
    assert torch.equal(again, terms) and torch.equal(hat2, hat)          # fixed summation order: bit for bit


def test_fused_terms_per_node_sweep():
    """One-atom graphs, each with its own s0: term 4 is one node's log p(h | z_0).  s0 from 1e-3 to 10 (the production value
    4 sigma_0 among them) x offsets of the true class from its centre from 0 to +-3 classes (exactly +-0.5, where one erff
    argument is 0, included) x three true classes, the other classes at their centres plus sigma_0 noise; and nodes 9
    classes away from every centre, where every class sits on the floor and the result is -log K.  Each node is held to
    float64 by C_SUM u sum|summands| plus the propagated erff term alone: the case-wide fp32 term of the sum bound is
    left out, so a fault confined to one regime is not hidden by the worst node of another."""
    K, nv, nb = 10, 4.0, 0.0
    s0_grid = torch.cat([torch.logspace(-3, 1, 41, dtype=torch.float64), torch.tensor([S0_PRODUCTION], dtype=torch.float64)])
    offs = torch.tensor([0.0, 0.125, 0.25, 0.4, 0.5, 0.6, 0.75, 1.0, 1.5, 2.0, 2.5, 3.0], dtype=torch.float64)
    offs = torch.cat([offs, -offs[1:]])
    ks = torch.tensor([0.0, 4.0, 9.0], dtype=torch.float64)
    S, O, Kk = torch.meshgrid(s0_grid, offs, ks, indexing='ij')
    S, O, Kk = S.flatten(), O.flatten(), Kk.flatten().long()
    n = S.numel()
    g = torch.Generator().manual_seed(77)
    un = torch.nn.functional.one_hot(Kk, K).double()
    noise = torch.randn((n, K), generator=g, dtype=torch.double) * (S / nv).unsqueeze(1) * (1 - un)
    un = un * (1 + O).unsqueeze(1) + noise
    floored = torch.arange(0, n, 50)                             # every 50th node: 9 classes above every centre
    un[floored] = 10.0
    wide = S[floored] <= 1.0
    floored = floored[wide]                                     # (with s0 > 1 nothing is 9 widths away)
    lm = torch.arange(n).cuda()
    pm = torch.zeros(1, dtype=torch.long).cuda()              # one pocket row: ignored by the ligand-only form
    xh = torch.cat([torch.zeros((n, 3), dtype=torch.double), torch.nn.functional.one_hot(Kk, K).double() / nv], 1)
    z0 = torch.cat([torch.zeros((n, 3), dtype=torch.double), un / nv], 1)
    f = lambda t: t.float().cuda().contiguous()
    zeros = torch.zeros((n, 3 + K))
    side_l = [f(xh), f(zeros), f(zeros), f(zeros), f(z0), f(zeros), f(zeros)]
    coef = torch.stack([torch.full((n,), 0.02236, dtype=torch.double), S, torch.ones(n, dtype=torch.double),
                        torch.zeros(n, dtype=torch.double)], 1).float().cuda().contiguous()
    rc, terms, hat = _launch_terms(side_l, None, lm, pm, coef, nv, nb, -1, K, K, n)
    assert rc == 0
    r64 = nc.vlb_terms_ref(side_l, None, lm, pm, coef, nv, nb, -1, n, torch.float64)
    r32 = nc.vlb_terms_ref(side_l, None, lm, pm, coef, nv, nb, -1, n, torch.float32)
    nc.assert_sum_bound(terms, r32, r64, 'sweep', TERM_NAMES)
    got = terms[:, 4].double().cpu()
    assert torch.isfinite(got).all()
    want, mag, slack = (x.cpu() for x in (r64.node_lig, r64.node_lig_mag, r64.node_lig_slack))
    err = (got - want).abs()
    bound = nc.C_SUM * nc.U32 * mag + slack
    bad = torch.nonzero(err > bound).flatten()
    assert bad.numel() == 0, (f'{bad.numel()} of {n} nodes outside their bound; first: s0 {float(S[bad[0]]):.4g} offset '
                              f'{float(O[bad[0]])} class {int(Kk[bad[0]])}: native {float(got[bad[0]])!r} float64 '
                              f'{float(want[bad[0]])!r} bound {float(bound[bad[0]]):.3e}')
    exact = slack == 0                                          # no class within reach of erff's rounding: pure fp32 rounding
    assert int(exact.sum()) > n // 10
    err32 = (r32.node_lig.double().cpu() - want).abs()
    print(f'sweep: {n} nodes, {int(exact.sum())} without erff slack; worst error / bound {float((err / bound).max()):.3f}; '
          f'largest error {float(err.max()):.3e} (fp32 restatement {float(err32.max()):.3e})')
    # every class floored: -log K to two ulp of |log 1e-10|
    assert floored.numel() > 20
    assert float((got[floored] + math.log(K)).abs().max()) <= 2 * 2.0 ** -19
    # the true class at its centre with the production s0: a probability of 1 up to the neighbours' tails (3e-7 in float64)
    sel = (S == S0_PRODUCTION) & (O == 0)
    sel[::50] = False
    assert float(got[sel].abs().max()) <= 1e-6


def test_argument_checks_launch_nothing():
    lib = _native.load()
    n_lig, n_poc, A, R = [4, 3], [5, 6], 10, 12
    lm, pm = _masks(n_lig, n_poc)
    side_l, side_p, coef = _production_sides(lm, pm, 2, A, R, 4.0, 0.0, torch.full((2,), S0_PRODUCTION), True,
                                             torch.Generator().manual_seed(1))

    def terms_call(side_l=side_l, side_p=side_p, coef=coef, lm=lm, A=A, R=R, nv=4.0, vnode=-1, n=2, out=True):
        terms = torch.full((2, 11), float('nan'), device='cuda')
        hat = torch.full_like(side_l[0], float('nan'))
        rc = lib.dsb_ddpm_vlb_terms(*[_ptr(x) for x in side_l], *[_ptr(x) for x in (side_p or [None] * 6)], _ptr(coef), _ptr(lm),
                                    _ptr(pm), len(side_l[0]), len(pm), n, A, R, nv, 0.0, vnode,
                                    _ptr(terms) if out else None, _ptr(hat), _stream())
        torch.cuda.synchronize()
        assert torch.isnan(terms).all() and torch.isnan(hat).all()      # nothing was launched
        return rc

    bad = {
        'null required input': dict(side_l=side_l[:3] + [None] + side_l[4:]),
        'null coef': dict(coef=None),
        'null mask': dict(lm=None),
        'null output': dict(out=False),
        'pocket without companions': dict(side_p=side_p[:2] + [None] + side_p[3:]),
        'vnode_idx >= atom_nf': dict(vnode=A),
        'norm_value_h <= 0': dict(nv=0.0),
        'norm_value_h nan': dict(nv=float('nan')),
        'atom_nf <= 0': dict(A=0),
        'residue_nf <= 0': dict(R=0),
    }
    for what, kw in bad.items():
        rc = terms_call(**kw)
        assert rc == -1, (what, rc)                                  # DSB_ERR_INVALID_ARGUMENT
        assert lib.dsb_last_error().decode(), what
    assert terms_call(n=0) == 0                                     # no graphs: success, nothing written

    xl, el, xp, ep = side_l[0], side_l[2], side_p[0], side_p[1]
    c2 = coef[:, 2:].contiguous()

    def noise_call(xl=xl, el=el, xp=xp, ep=ep, c2=c2, n=2, zp=True):
        zl = torch.full_like(side_l[0], float('nan'))
        zpo = torch.full_like(side_p[0], float('nan'))
        rc = lib.dsb_ddpm_noise(_ptr(xl), _ptr(el), _ptr(xp), _ptr(ep), _ptr(c2), _ptr(lm), _ptr(pm), len(lm), len(pm), n, A, R,
                                _ptr(zl), _ptr(zpo) if zp else None, _stream())
        torch.cuda.synchronize()
        assert torch.isnan(zl).all() and torch.isnan(zpo).all()
        return rc

    for what, kw in {'null ligand': dict(xl=None), 'null noise': dict(el=None), 'null coef': dict(c2=None),
                     'pocket without its noise': dict(ep=None), 'pocket without its output': dict(zp=False)}.items():
        assert noise_call(**kw) == -1, what
        assert lib.dsb_last_error().decode(), what
    assert noise_call(n=0) == 0


# ---- b. noising at every timestep ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('variant', ['joint', 'simple', 'conditional'])
def test_noising_at_every_timestep(variant):
    """501 ragged graphs, graph g at t = g / 500 of polynomial_2 (precision 5e-4), one launch: dsb_ddpm_noise (joint, simple)
    or dsb_ddpm_ligand_update with coef = (1 / alpha, 0, sigma) (conditional), coefficients built as the forward builds
    them, against float64 alpha xh + sigma eps from the same fp32 table; the ligand COM of the conditional result is zero
    within the bound."""
    T = 500
    cfg = JOINT_CFG if variant == 'joint' else DDPM_CFG
    A, R = cfg.atom_nf, cfg.residue_nf
    n = T + 1
    g = torch.Generator().manual_seed(5)
    n_lig = (torch.randint(1, 12, (n,), generator=g)).tolist()
    n_poc = (torch.randint(0, 30, (n,), generator=g)).tolist()
    n_lig[7], n_poc[3] = 140, 300                               # more rows than one block has threads
    lm, pm = _masks(n_lig, n_poc)
    spec = dict(model=variant, T=T, schedule='polynomial_2', seed=0)
    ddpm = base._build(spec, 'cuda', native=True, cfg=cfg)
    xl = torch.cat([torch.randn((len(lm), 3), generator=g) * 3, torch.randn((len(lm), A), generator=g).sign() / 4], 1).cuda()
    xp = torch.cat([torch.randn((len(pm), 3), generator=g) * 8, torch.randn((len(pm), R), generator=g).sign() / 4], 1).cuda()
    el, ep = torch.randn((len(lm), 3 + A), generator=g).cuda(), torch.randn((len(pm), 3 + R), generator=g).cuda()
    t_int = torch.arange(n, device='cuda')
    gamma = ddpm.inflate_batch_array(ddpm.gamma(t_int.float().view(n, 1) / T), xl)
    if variant == 'joint':
        z, zp = ddpm._native_noise(xl, el, xp, ep, lm, pm, gamma)
    else:
        z, zp = ddpm._native_noise_conditional(xl, el, xp, lm, pm, gamma)
    torch.cuda.synchronize()
    ref = {}
    for dtype in (torch.float32, torch.float64):
        gam = nc.gamma_of(ddpm, t_int, dtype)
        ref[dtype] = nc.noise_ref(variant, xl, el, xp, ep, lm, pm, nc.alpha_of(gam), nc.sigma_of(gam), n, dtype)
    r32, r64 = ref[torch.float32], ref[torch.float64]
    ratio = nc.assert_element_bound(z, r32[0], r64[0], r64[2], f'{variant} z_lig')
    if variant == 'joint':
        a, s = nc.alpha_of(nc.gamma_of(ddpm, t_int, torch.float64))[pm, None], nc.sigma_of(nc.gamma_of(ddpm, t_int, torch.float64))[pm, None]
        nc.assert_element_bound(zp, r32[1], r64[1], (a * xp).abs() + (s * ep).abs(), 'joint z_pocket')
    elif variant == 'simple':
        assert zp is xp or torch.equal(zp, xp)
    else:
        shift = nc.seg_sum(r64[2][:, :3], lm, n) / torch.tensor(n_lig, device='cuda').clamp(min=1)[:, None]
        scale = xp.double().abs()
        scale[:, :3] += shift[pm]
        nc.assert_element_bound(zp, r32[1], r64[1], scale, 'conditional pocket')
        com = nc.seg_sum(z[:, :3].double(), lm, n) / torch.tensor(n_lig, device='cuda')[:, None]
        assert bool((com.abs() <= nc.C_EL * nc.U32 * shift.clamp(min=1e-30)).all()), float(com.abs().max())
    print(f'{variant}: z_lig error / bound {ratio:.3f} over t = 0 .. {T}')


# ---- c, d. the forward, stage by stage ---------------------------------------------------------------------------------------
def _check_forward(kind, ddpm, hist, ligand, pocket, rec, out, what):
    """Every stage of one recorded native forward against float64, each fed the fp32 inputs the native stage received.
    Returns (Restated float64 on the native stage inputs, {stage: worst error / bound})."""
    ratios = {}
    t_int = out[10]
    eps_t, eps_0 = rec.eps(kind)
    (args_t, z_t), (args_0, z_0) = rec.noisings()
    xh0 = (args_t[0], args_t[2])
    z = ([z_t[0], z_t[1]], [z_0[0], z_0[1]])
    R = {dt: nc.restate_forward(kind, ddpm, hist, ligand, pocket, t_int, eps_t, eps_0, rec.nets(), dt, xh0=xh0, z=z)
         for dt in (torch.float32, torch.float64)}
    r32, r64 = R[torch.float32], R[torch.float64]
    # centring and normalisation of the inputs
    raw = nc.centred_inputs(kind, ddpm, ligand, pocket, torch.float64)
    n = len(ligand['size'])
    mean_abs = lambda part: nc.seg_sum(part['x'].double().abs(), part['mask'], n) / part['size'].clamp(min=1)[:, None]
    spread = mean_abs(ligand) + mean_abs(pocket)               # a centre of mass errs by u times the mean |x| it averages
    for got, want, part in ((xh0[0], raw[0], ligand), (xh0[1], raw[1], pocket)):
        scale = torch.cat([part['x'].double().abs() + spread[part['mask']], want[:, 3:].abs()], 1)
        assert bool(((got.double() - want).abs() <= nc.C_SUM * nc.U32 * scale + 1e-30).all()), what + ' centred inputs'
    # noising (the denoiser's inputs are these very tensors)
    for tag, got, a, b, call in (('z_t', z_t, r32.z_t, r64.z_t, rec.dyn[0]), ('z_0', z_0, r32.z_0, r64.z_0, rec.dyn[1])):
        ratios[tag] = nc.assert_element_bound(got[0], a[0], b[0], b[2], f'{what} {tag}')
        assert torch.equal(call[0][0], got[0]) and torch.equal(call[0][1], got[1])
        if kind == 'joint':
            assert float((got[1].double() - b[1]).abs().max()) <= max(2 * float((a[1].double() - b[1]).abs().max()),
                                                                    nc.C_EL * nc.U32 * float(b[1].abs().max()))
    # the eleven sums and xh_lig_hat from the recorded denoiser outputs
    (_, (terms, hat)), = rec.terms_calls
    ratios['terms'] = nc.assert_sum_bound(terms, r32.terms, r64.terms, what, TERM_NAMES)
    ratios['xh_lig_hat'] = nc.assert_element_bound(hat, r32.terms.hat, r64.terms.hat, r64.terms.hat_scale, what + ' xh_lig_hat')
    assert torch.equal(out[11], hat)
    # the per-graph scalar algebra: every entry of the return tuple, per complex
    mag = r64.terms.mag
    sigma_T = nc.sigma_of(r64.gamma['T'])
    dof = (r64.out['neg_log_constants'] / (0.5 * r64.gamma['0'] + 0.5 * math.log(2 * math.pi))).abs()
    scales = {'kl_prior': (dof + 1) * (sigma_T.log().abs() + 0.5 * sigma_T ** 2 + 0.5) + 0.5 * (mag[:, 5] + mag[:, 6]),
              'SNR_weight': 1 + (1 - r64.out['SNR_weight']).abs(),       # 1 - exp(.): an absolute error of u in either addend
              'error_t_lig': mag[:, 0], 'error_t_pocket': mag[:, 1], 'loss_0_x_ligand': mag[:, 2], 'loss_0_x_pocket': mag[:, 3]}
    for key, got in zip(RETURN_NAMES[:-2], out[:-3]):
        want64, want32 = r64.out[key], r32.out[key]
        if key == 'loss_0_h':                                   # the terms check above held it with the erff slack
            continue
        if want64.dim() == 0:
            assert float(got) == 0.0, key
            continue
        scale = scales.get(key, want64.abs())
        ratios[key] = nc.assert_scalar_bound(got, want32, want64, scale, f'{what} {key}')
    assert torch.equal(out[10].cpu().double(), r64.out['t_int'].cpu())
    for k, v in out[-1].items():
        ratios['info ' + k] = nc.assert_scalar_bound(v, r32.info[k], r64.info[k], r64.info[k].abs(), f'{what} info {k}')
    assert sorted(out[-1]) == sorted(r64.info)
    return r32, r64, ratios


def _sweep_batch(cfg, n, seed):
    g = torch.Generator().manual_seed(seed)
    n_lig = torch.randint(3, 10, (n,), generator=g).tolist()
    n_poc = torch.randint(6, 21, (n,), generator=g).tolist()
    data = syn.synthetic_complex_batch(cfg, n_lig, n_poc, seed=seed)
    ligand = {'x': data['lig_coords'], 'one_hot': data['lig_one_hot'], 'size': data['num_lig_atoms'], 'mask': data['lig_mask']}
    pocket = {'x': data['pocket_coords'], 'one_hot': data['pocket_one_hot'], 'size': data['num_pocket_nodes'],
              'mask': data['pocket_mask']}
    return ({k: v.cuda() for k, v in ligand.items()}, {k: v.cuda() for k, v in pocket.items()})


SWEEP = [('conditional', False, '3xfp16', 'polynomial_2'), ('conditional', True, '3xfp16', 'polynomial_2'),
         ('simple', False, '3xfp16', 'polynomial_2'), ('joint', False, '3xfp16', 'polynomial_2'),
         ('conditional', False, '3xtf32', 'polynomial_2'), ('joint', False, 'fp32', 'polynomial_2'),
         ('conditional', False, '3xfp16', 'learned')]


@pytest.mark.parametrize('kind,vnode,math_mode,schedule', SWEEP)
def test_forward_at_every_timestep(kind, vnode, math_mode, schedule):
    """500 small ragged complexes, complex g evaluated at t = g + 1 of T = 500 (t = 1: s = 0 and SNR_weight from
    gamma_0 - gamma_1; t = T: alpha_T = 0.022 in the noising and in xh_lig_hat), H = 128."""
    T = 500
    cfg = (JOINT_CFG if kind == 'joint' else DDPM_CFG).with_(hidden_nf=128)
    spec = dict(model=kind, T=T, schedule=schedule, seed=0, vnode=vnode, n_lig=None)
    ddpm = base._build(spec, 'cuda', native=True, cfg=cfg, math_mode=math_mode)
    ddpm.dynamics.deterministic = True
    assert ddpm._vlb_native('cuda')
    ligand, pocket = _sweep_batch(cfg, T, seed=17)
    if vnode:
        ligand['one_hot'][::4] = 0
        ligand['one_hot'][::4, cfg.atom_nf - 1] = 1
    t_inject = torch.arange(1, T + 1)
    copy = lambda part: {k: v.clone() for k, v in part.items()}
    torch.manual_seed(3)
    with nc.ForwardRecorder(ddpm, t_inject) as rec:
        out = ddpm(copy(ligand), copy(pocket), return_info=True)
    torch.manual_seed(3)
    randint, torch.randint = torch.randint, (lambda lo, hi, size, device=None: t_inject.view(size).to(device))
    try:
        plain = ddpm(copy(ligand), copy(pocket), return_info=True)
    finally:
        torch.randint = randint
    for a, b in zip(out[:-1], plain[:-1]):                      # the recorder ran the production path: bit for bit
        assert torch.equal(a, b)
    assert all(torch.equal(out[-1][k], plain[-1][k]) for k in out[-1])
    _, r64, ratios = _check_forward(kind, ddpm, NLL_HIST, ligand, pocket, rec, out, f'{kind} vnode={vnode} {math_mode} {schedule}')
    assert float(out[3][0]) < 0 and out[10].tolist() == list(range(1, T + 1))
    print(f'{kind} vnode={vnode} {math_mode} {schedule}: worst error / bound per stage '
          f'{ {k: (round(max(v), 3) if isinstance(v, list) else round(v, 3)) for k, v in ratios.items()} }')


def _nll_report(tag, nll, info, r32, r64, T, virtual_nodes=False):
    want, want_info, _, _ = nc.facade(r64.out, r64.info, T, virtual_nodes)
    want32, info32, _, _ = nc.facade(r32.out, r32.info, T, virtual_nodes)
    err = (nll.double() - want).abs()
    err32 = (want32.double() - want).abs()
    # nll is a sum of terms of both signs: its honest scale is the sum of their magnitudes
    scale = sum(r64.out[k].abs() for k in ('loss_0_x_ligand', 'loss_0_x_pocket', 'loss_0_h', 'neg_log_constants', 'kl_prior',
                                           'delta_log_px', 'log_pN')) \
        + T * 0.5 * r64.out['SNR_weight'].abs() * (r64.out['error_t_lig'] + r64.out['error_t_pocket'])
    ratio = nc.assert_scalar_bound(nll, want32, want, scale + r64.terms.slack[:, 4] / (nc.C_SUM * nc.U32), tag + ' nll')
    for k in info:
        nc.assert_scalar_bound(info[k], info32[k], want_info[k], want_info[k].abs() + 1e-3, f'{tag} info {k}')
    assert not info or sorted(info) == sorted(want_info)
    print(f'{tag}: [{_card()}] nll per complex: mean |nll| {float(want.abs().mean()):.1f}, native |error| max {float(err.max()):.3e} '
          f'mean {float(err.mean()):.3e}; fp32 restatement max {float(err32.max()):.3e}; err_native / err_fp32 (max) '
          f'{float(err.max() / err32.max().clamp(min=1e-300)):.2f}; error / bound {ratio:.3f}')
    return err, err32


@pytest.mark.parametrize('math_mode,deterministic', [('3xfp16', True), ('auto', False), ('3xtf32', False), ('fp32', False)])
def test_production_nll_conditional(math_mode, deterministic):
    """LigandPocketDDPM.forward on the configs[2] batch (64 x (25 + 175), H = 256, 6 layers, T = 500 polynomial_2)."""
    model, cfg = base._full_model()
    model.ddpm.dynamics.math_mode = math_mode
    model.ddpm.dynamics.deterministic = deterministic
    data = syn.synthetic_complex_batch(cfg, [25] * 64, [175] * 64, seed=3)
    ligand, pocket = model.get_ligand_and_pocket(data)
    t_inject = torch.cat([torch.tensor([1, 500]), torch.randint(1, 501, (62,), generator=torch.Generator().manual_seed(2))])
    torch.manual_seed(7)
    with nc.ForwardRecorder(model.ddpm, t_inject) as rec:
        nll, info = model(data)
    hist = np.ones((27, 177)).tolist()
    tag = f'configs[2] {math_mode} deterministic={deterministic}'
    r32, r64, ratios = _check_forward('conditional', model.ddpm, hist, ligand, pocket, rec, rec.out, tag)
    print(f'{tag}: err_native / bound per term {[round(x, 3) for x in ratios["terms"]]}')
    _nll_report(tag, nll, info, r32, r64, 500)
    if deterministic:
        torch.manual_seed(7)
        with nc.ForwardRecorder(model.ddpm, t_inject):
            again, _ = model(data)
        assert torch.equal(again, nll)


def test_production_nll_joint():
    """EnVariationalDiffusion.forward of the joint production configuration (H = 128, 5 layers, update_pocket_coords) on
    16 x (25 + 175), T = 500, default math mode, deterministic; nll assembled as the facade assembles it."""
    cfg = FULLATOM_JOINT
    spec = dict(model='joint', T=500, schedule='polynomial_2', seed=0, n_lig=None)
    ddpm = base._build(spec, 'cuda', native=True, cfg=cfg)
    hist = np.ones((27, 177)).tolist()
    ddpm.size_distribution = type(ddpm.size_distribution)(hist)
    ddpm.dynamics.deterministic = True
    data = syn.synthetic_complex_batch(cfg, [25] * 16, [175] * 16, seed=3)
    ligand = {'x': data['lig_coords'].cuda(), 'one_hot': data['lig_one_hot'].cuda(), 'size': data['num_lig_atoms'].cuda(),
              'mask': data['lig_mask'].cuda()}
    pocket = {'x': data['pocket_coords'].cuda(), 'one_hot': data['pocket_one_hot'].cuda(),
              'size': data['num_pocket_nodes'].cuda(), 'mask': data['pocket_mask'].cuda()}
    t_inject = torch.cat([torch.tensor([1, 500]), torch.randint(1, 501, (14,), generator=torch.Generator().manual_seed(4))])
    copy = lambda part: {k: v.clone() for k, v in part.items()}
    torch.manual_seed(11)
    with nc.ForwardRecorder(ddpm, t_inject) as rec:
        out = ddpm(copy(ligand), copy(pocket), return_info=True)
    r32, r64, ratios = _check_forward('joint', ddpm, hist, ligand, pocket, rec, out, 'joint production')
    print(f'joint production: err_native / bound per term {[round(x, 3) for x in ratios["terms"]]}')
    named = dict(zip(RETURN_NAMES, out[:-1]))
    nll, info, _, _ = nc.facade({k: v for k, v in named.items()}, out[-1], 500, False)
    _nll_report('joint production', nll, {}, r32, r64, 500)
