"""float64 restatement of the eval-mode variational bound (validation / test NLL), and the bounds the tests hold the native
path to.

Every function takes a ``dtype``: float64 is the truth, float32 the yardstick (the same formulas in the precision the
kernels work in).  The formulas are written from the reference, not by calling this repo's loss code:

  noising              z = alpha x + sigma eps                   en_diffusion.py:302-317, conditional_model.py:140-183
  error_t, loss_0_x    sums of (eps - net)^2                     en_diffusion.py:385-390, :185-215, conditional_model.py:58-110
  log p(h | z_0)       discretised Gaussian, +1e-10, logsumexp   en_diffusion.py:216-255, :949
  kl_prior             gaussian_KL of alpha_T xh against N(0, 1) en_diffusion.py:109-155, :840-853, conditional_model.py:20-56
  constants            delta_log_px, log_constants_p_x_given_z0  en_diffusion.py:171-183, :332-334
  schedule             alpha, sigma, SNR, polynomial_2, gamma    en_diffusion.py:865-878, :1125-1190, :1064-1102
  size prior           log p(N), log p(N_lig | N_pocket)         en_diffusion.py:1002-1019
  xh_lig_hat           z_t / alpha_t - net sigma_t / alpha_t     en_diffusion.py:471-477
  facade               loss_t, loss_0, nll, info means           lightning_modules.py:236-302

Bounds, chosen once for every case (u = 2^-24, the unit roundoff of float32):

  element   |native - f64| <= max(R |f32 - f64|_max over the tensor, C_EL u scale), scale = sum of |addends| of the element
  sum       |native - f64| <= max(R |f32 - f64|_max over the case, C_SUM u sum|summands|) per graph and term
  term 4    the sum bound plus the propagated error of erff: each class probability p_c carries an absolute error
            delta_c = C_ERF u (1 + (|c| + 1/2) / s0 (phi(hi) + phi(lo))) (erff to 2 ulp, and the rounding of its argument
            times the slope of Phi); where both erff arguments are beyond 4 on the same side erff is exactly +-1 in fp32, p_c
            is exactly the 1e-10 floor, and delta_c is the tail mass float64 still sees (up to 8e-9, zero far out);
            log p_c then moves by at most
            log((p_c + delta_c) / max(p_c - delta_c, 1e-10)) and the log-sum-exp by the same expression of the sums.
            Without this term no fp32 evaluation can be held to float64 where p_c is a few multiples of 2^-25: one ulp
            of erff's argument (torch divides by sqrt 2 by multiplying with its rounded reciprocal, the kernel divides)
            changes p_c by a factor there, which is the operation's conditioning, not an error of either evaluation.

  R = 2, C_EL = 8, C_SUM = 16, C_ERF = 4.  Measured on an H100 the largest ratio error / bound of each test is printed
  by the GPU tests (see DESIGN.md section 10 for the production-size figures).
"""
import math

import numpy as np
import torch

U32 = 2.0 ** -24
R_FP32, C_EL, C_SUM, C_ERF = 2.0, 8.0, 16.0, 4.0
SQRT2 = math.sqrt(2.0)

# Two more likelihood goldens at the production schedule (T = 500, polynomial_2, precision 5e-4): the timestep draw is
# injected so that one batch of four complexes holds t = 1, t = T and two interior steps.
NLL_T500_CASES = {
    't500_cond': dict(model='conditional', n_lig=[7, 5, 6, 4], T=500, schedule='polynomial_2', seed=311),
    't500_joint': dict(model='joint', n_lig=[6, 4, 5, 7], T=500, schedule='polynomial_2', seed=312),
}
T500_STEPS = [1, 500, 137, 420]
T500_POCKET = [22, 17, 9, 25]


def seg_sum(v, mask, n):
    out = torch.zeros((n,) + tuple(v.shape[1:]), dtype=v.dtype, device=v.device)
    return out.index_add_(0, mask, v)


# ---- the schedule -----------------------------------------------------------------------------------------------------
def polynomial_gamma64(timesteps, precision, power=2.0):
    """gamma[0..T] of the polynomial schedule in float64 (en_diffusion.py:1125-1190): alpha^2 = (1 - (x / steps)^power)^2,
    ratios alpha_t^2 / alpha_{t-1}^2 clipped to [0.001, 1], squeezed to [precision, 1 - precision]."""
    steps = timesteps + 1
    x = np.linspace(0, steps, steps)
    a2 = (1.0 - np.power(x / steps, power)) ** 2
    ext = np.concatenate([np.ones(1), a2])
    a2 = np.cumprod(np.clip(ext[1:] / ext[:-1], a_min=0.001, a_max=1.0))
    a2 = (1.0 - 2.0 * precision) * a2 + precision
    return -(np.log(a2) - np.log(1.0 - a2))


def gamma_network(sd, t, dtype):
    """The learned schedule (en_diffusion.py:1031-1102) evaluated in ``dtype`` from its stored weights."""
    p = {k: v.detach().to(t.device, dtype) for k, v in sd.items()}
    lin = lambda x, name: torch.nn.functional.linear(x, torch.nn.functional.softplus(p[name + '.weight']), p[name + '.bias'])

    def tilde(x):
        a = lin(x, 'l1')
        return a + lin(torch.sigmoid(lin(a, 'l2')), 'l3')

    t = t.to(dtype).view(-1, 1)
    g0, g1, gt = tilde(torch.zeros_like(t)), tilde(torch.ones_like(t)), tilde(t)
    return (p['gamma_0'] + (p['gamma_1'] - p['gamma_0']) * (gt - g0) / (g1 - g0)).view(-1)


def gamma_of(ddpm, t_int, dtype):
    """gamma at the integer steps ``t_int`` [n] in ``dtype``: the stored table (a checkpoint's fp32 parameter is the
    schedule; its distance from the float64 formula is pinned by the CPU test) or the learned network."""
    t_int = t_int.view(-1)
    if hasattr(ddpm.gamma, 'l1'):
        return gamma_network(ddpm.gamma.state_dict(), t_int.to(dtype) / ddpm.T, dtype)
    return ddpm.gamma.gamma.detach().to(t_int.device)[t_int.long()].to(dtype)


def alpha_of(gamma):
    return torch.sqrt(torch.sigmoid(-gamma))


def sigma_of(gamma):
    return torch.sqrt(torch.sigmoid(gamma))


# ---- noising ----------------------------------------------------------------------------------------------------------
def noise_ref(variant, xh_lig, eps_lig, xh_pocket, eps_pocket, lm, pm, alpha, sigma, n, dtype):
    """q(z_t | x, h) in ``dtype`` for 'joint' (eps.x already COM-free), 'simple' (ligand only, no projection) and
    'conditional' (ligand COM of z removed from z and from the pocket).  alpha, sigma: [n].  Returns z_lig, the pocket
    (noised, unchanged or shifted) and the per-element scale of z_lig (sum of the magnitudes of its addends)."""
    d = lambda x: None if x is None else x.to(dtype)
    xh_lig, eps_lig, xh_pocket, eps_pocket, alpha, sigma = map(d, (xh_lig, eps_lig, xh_pocket, eps_pocket, alpha, sigma))
    a, s = alpha[lm].unsqueeze(1), sigma[lm].unsqueeze(1)
    z = a * xh_lig + s * eps_lig
    scale = (a * xh_lig).abs() + (s * eps_lig).abs()
    if variant == 'joint':
        return z, alpha[pm].unsqueeze(1) * xh_pocket + sigma[pm].unsqueeze(1) * eps_pocket, scale
    if variant == 'simple':
        return z, xh_pocket, scale
    cnt = seg_sum(torch.ones_like(z[:, 0]), lm, n).clamp(min=1).unsqueeze(1)
    com = seg_sum(z[:, :3], lm, n) / cnt
    scale = scale.clone()
    scale[:, :3] += (seg_sum(scale[:, :3], lm, n) / cnt)[lm]
    z = torch.cat([z[:, :3] - com[lm], z[:, 3:]], 1)
    pocket = torch.cat([xh_pocket[:, :3] - com[pm], xh_pocket[:, 3:]], 1)
    return z, pocket, scale


# ---- the eleven per-graph terms ---------------------------------------------------------------------------------------
def log_ph_nodes(z0_h, one_hot_h, s0_rows, nv, nb, dtype):
    """log p(h | z_0) of every node (en_diffusion.py:216-255).  Returns the node values, the magnitude of their summands
    and the propagated erff slack of the module docstring (meaningful in float64)."""
    z0_h, one_hot_h, w = z0_h.to(dtype), one_hot_h.to(dtype), s0_rows.to(dtype).view(-1, 1)
    target = one_hot_h * nv + nb
    ctr = (z0_h * nv + nb) - 1
    cdf = lambda v: 0.5 * (1. + torch.erf(v / SQRT2))
    hi, lo = (ctr + 0.5) / w, (ctr - 0.5) / w
    mass = cdf(hi) - cdf(lo)
    p = mass + 1e-10
    lp = torch.log(p)
    logz = torch.logsumexp(lp, dim=1, keepdim=True)
    node = ((lp - logz) * target).sum(1)
    mag = (target.abs() * (1 + lp.abs() + logz.abs())).sum(1)
    phi = lambda v: torch.exp(-0.5 * v * v) / math.sqrt(2 * math.pi)
    saturated = (hi.abs() > 4 * SQRT2) & (lo.abs() > 4 * SQRT2) & (hi.sign() == lo.sign())
    delta = C_ERF * U32 * (1 + (ctr.abs() + 0.5) / w * (phi(hi) + phi(lo)))
    delta = torch.where(saturated, mass.abs(), delta)
    e = torch.log((p + delta) / (p - delta).clamp(min=1e-10))
    z_sum, d_sum = p.sum(1, keepdim=True), delta.sum(1, keepdim=True)
    e_z = torch.log((z_sum + d_sum) / (z_sum - d_sum).clamp(min=1e-10 * p.shape[1]))
    slack = (target.abs() * (e + e_z)).sum(1)
    return node, mag, slack


class Terms:
    """terms [n, 11], xh_lig_hat, its per-element scale, mag [n, 11] = sum |summands|, slack [n, 11] (erff, column 4 only),
    node_lig = log p(h | z_0) per ligand node (with its mag and slack)."""


def vlb_terms_ref(lig_side, pocket_side, lm, pm, coef, nv, nb, vnode, n, dtype):
    """dsb_ddpm_vlb_terms restated in ``dtype``, column for column as include/diffsbdd_b200.h lists them.
    lig_side = (xh0, z_t, eps_t, net_t, z_0, eps_0, net_0), pocket_side = (xh0, eps_t, net_t, z_0, eps_0, net_0) or None,
    coef [n, 4] = (alpha_T, sigma_0 norm_value_h, alpha_t, sigma_t) as the kernel receives it (fp32 values)."""
    d = lambda x: x.to(dtype)
    xl, ztl, etl, ntl, z0l, e0l, n0l = map(d, lig_side)
    coef = d(coef)
    aT, s0, at, st = (coef[:, k] for k in range(4))
    out = Terms()
    terms = torch.zeros((n, 11), dtype=dtype, device=xl.device)
    mag = torch.zeros_like(terms)
    slack = torch.zeros_like(terms)

    def put(k, v, mask, add=False):
        s = seg_sum(v, mask, n)
        terms[:, k] = terms[:, k] + s if add else s
        mag[:, k] = mag[:, k] + seg_sum(v.abs(), mask, n) if add else seg_sum(v.abs(), mask, n)

    sq_t, sq_0 = (etl - ntl) ** 2, (e0l[:, :3] - n0l[:, :3]) ** 2
    if vnode >= 0:                                    # conditional_model.py:76-78, :264-266: x of virtual atoms left out
        virt = xl[:, 3 + vnode] != 0
        sq_t, sq_0 = sq_t.clone(), sq_0.clone()
        sq_t[virt, :3] = 0
        sq_0[virt] = 0
    put(0, sq_t.sum(1), lm)
    put(2, sq_0.sum(1), lm)
    node, nmag, nslack = log_ph_nodes(z0l[:, 3:], xl[:, 3:], s0[lm], nv, nb, dtype)
    out.node_lig, out.node_lig_mag, out.node_lig_slack = node, nmag, nslack
    terms[:, 4], mag[:, 4], slack[:, 4] = seg_sum(node, lm, n), seg_sum(nmag, lm, n), seg_sum(nslack, lm, n)
    mu = aT[lm].unsqueeze(1) * xl
    put(5, (mu[:, :3] ** 2).sum(1), lm)
    put(6, (mu[:, 3:] ** 2).sum(1), lm)
    put(7, ntl[:, :3].abs().sum(1), lm)
    put(8, ntl[:, 3:].abs().sum(1), lm)
    if pocket_side is not None:
        xp, etp, ntp, z0p, e0p, n0p = map(d, pocket_side)
        put(1, ((etp - ntp) ** 2).sum(1), pm)
        put(3, ((e0p[:, :3] - n0p[:, :3]) ** 2).sum(1), pm)
        node, nmag, nslack = log_ph_nodes(z0p[:, 3:], xp[:, 3:], s0[pm], nv, nb, dtype)
        terms[:, 4] += seg_sum(node, pm, n)
        mag[:, 4] += seg_sum(nmag, pm, n)
        slack[:, 4] += seg_sum(nslack, pm, n)
        mu = aT[pm].unsqueeze(1) * xp
        put(5, (mu[:, :3] ** 2).sum(1), pm, add=True)
        put(6, (mu[:, 3:] ** 2).sum(1), pm, add=True)
        put(9, ntp[:, :3].abs().sum(1), pm)
        put(10, ntp[:, 3:].abs().sum(1), pm)
    a, s = at[lm].unsqueeze(1), st[lm].unsqueeze(1)
    out.hat = ztl / a - ntl * s / a
    out.hat_scale = (ztl / a).abs() + (ntl * s / a).abs()
    out.terms, out.mag, out.slack = terms, mag, slack
    return out


# ---- per-graph scalar algebra -----------------------------------------------------------------------------------------
def log_pn_numpy(histogram, n_lig, n_pocket, conditional):
    """log p(N_lig, N_pocket) or log p(N_lig | N_pocket) from the size histogram (en_diffusion.py:958-1019), in float64.
    The module keeps the table as float32 (histogram + 1e-3, normalised); this starts from the same float32 table."""
    hist = (torch.tensor(histogram).float() + 1e-3)
    p = (hist / hist.sum()).double().numpy()
    a, b = np.asarray(n_lig), np.asarray(n_pocket)
    joint = p[a, b] / p.sum()
    return np.log(joint / (p[:, b].sum(0) / p.sum())) if conditional else np.log(joint)


def scalar_algebra(terms, gamma_s, gamma_t, gamma_0, gamma_T, dof, norm_value_x, log_pn, n_lig, n_pocket, atom_nf,
                   residue_nf, conditional, dtype):
    """From the eleven per-graph sums to the return tuple of the DDPM ``forward`` (without t_int and xh_lig_hat) and its
    ``info`` means, in ``dtype``.  dof [n] = degrees of freedom of x (en_diffusion.py:914-916, conditional_model.py:713)."""
    d = lambda x: torch.as_tensor(x).to(dtype)
    terms, gamma_s, gamma_t, gamma_0, gamma_T, dof = map(d, (terms, gamma_s, gamma_t, gamma_0, gamma_T, dof))
    out = {'delta_log_px': -dof * math.log(norm_value_x),                                  # en_diffusion.py:332-334
           'error_t_lig': terms[:, 0], 'error_t_pocket': terms[:, 1],
           'SNR_weight': 1 - torch.exp(-(gamma_s - gamma_t)),                                # :375, :876-878
           'loss_0_x_ligand': 0.5 * terms[:, 2], 'loss_0_x_pocket': 0.5 * terms[:, 3], 'loss_0_h': -terms[:, 4],
           'neg_log_constants': -(dof * (-0.5 * gamma_0 - 0.5 * math.log(2 * math.pi)))}    # :171-183
    sigma_T = sigma_of(gamma_T)

    def kl(mu2, dim):                                                                        # :840-853 against N(0, I)
        return dim * torch.log(1 / sigma_T) + 0.5 * (dim * sigma_T ** 2 + mu2) / 1.0 - 0.5 * dim

    out['kl_prior'] = kl(terms[:, 5], dof) + kl(terms[:, 6], torch.ones_like(dof))        # :109-155
    out['log_pN'] = d(log_pn)
    if conditional:
        out['error_t_pocket'] = out['loss_0_x_pocket'] = torch.zeros((), dtype=dtype)
    cl, cp = d(n_lig).clamp(min=1), d(n_pocket).clamp(min=1)
    info = {'eps_hat_lig_x': (terms[:, 7] / (3 * cl)).mean(), 'eps_hat_lig_h': (terms[:, 8] / (atom_nf * cl)).mean()}
    if not conditional:
        info['eps_hat_pocket_x'] = (terms[:, 9] / (3 * cp)).mean()
        info['eps_hat_pocket_h'] = (terms[:, 10] / (residue_nf * cp)).mean()
    return out, info


def facade(out, info, T, virtual_nodes):
    """LigandPocketDDPM.forward (lightning_modules.py:236-302, the VLB / evaluation branch): nll per complex and the
    batch means added to ``info``."""
    loss_t = -T * 0.5 * out['SNR_weight'] * (out['error_t_lig'] + out['error_t_pocket'])
    loss_0 = out['loss_0_x_ligand'] + out['loss_0_x_pocket'] + out['loss_0_h'] + out['neg_log_constants']
    nll = loss_t + loss_0 + out['kl_prior'] - out['delta_log_px']
    if not virtual_nodes:
        nll = nll - out['log_pN']
    info = dict(info)
    for key, val in (('error_t_lig', out['error_t_lig']), ('error_t_pocket', out['error_t_pocket']),
                     ('SNR_weight', out['SNR_weight']), ('loss_0', loss_0), ('kl_prior', out['kl_prior']),
                     ('delta_log_px', out['delta_log_px']), ('neg_log_const_0', out['neg_log_constants']),
                     ('log_pN', out['log_pN'])):
        info[key] = val.mean(0)
    return nll, info, loss_t, loss_0


# ---- bounds -----------------------------------------------------------------------------------------------------------
def _f64(x):
    return x.detach().cpu().double()


def assert_element_bound(got, ref32, ref64, scale64, what):
    """Element-wise bound of the module docstring.  Returns error / bound of the worst element."""
    got, ref32, ref64, scale64 = map(_f64, (got, ref32, ref64, scale64))
    assert torch.isfinite(got).all(), f'{what}: non-finite output'
    err = (got - ref64).abs()
    bound = torch.maximum(torch.full_like(err, R_FP32 * float((ref32 - ref64).abs().max()) if err.numel() else 0.0),
                          C_EL * U32 * scale64)
    bad = err > bound
    i = int(torch.argmax(err - bound)) if err.numel() else 0
    assert not bad.any(), (f'{what}: {int(bad.sum())} elements outside the bound, worst at flat index {i}: '
                           f'error {float(err.flatten()[i]):.3e} > {float(bound.flatten()[i]):.3e}')
    return float((err / bound.clamp(min=1e-300)).max()) if err.numel() else 0.0


def assert_sum_bound(got, ref32, ref64, what, names=None):
    """Per-graph, per-term bound of the module docstring.  got [n, k]; ref32 / ref64: Terms.  Returns the worst
    error / bound per term."""
    g, t32, t64, mag, slack = map(_f64, (got, ref32.terms, ref64.terms, ref64.mag, ref64.slack))
    assert torch.isfinite(g).all(), f'{what}: non-finite terms'
    err = (g - t64).abs()
    err32 = (t32 - t64).abs().max(dim=0, keepdim=True).values
    bound = torch.maximum(R_FP32 * err32.expand_as(err), C_SUM * U32 * mag) + slack
    bad = err > bound
    if bad.any():
        gi, k = [int(v) for v in torch.nonzero(bad)[0]]
        raise AssertionError(f'{what}: term {k if names is None else names[k]} of graph {gi}: native {float(g[gi, k])!r}, '
                             f'float64 {float(t64[gi, k])!r}, error {float(err[gi, k]):.3e} > bound {float(bound[gi, k]):.3e} '
                             f'(fp32 restatement {float(err32[0, k]):.3e}; {int(bad.sum())} entries outside)')
    return (err / bound.clamp(min=1e-300)).max(dim=0).values.tolist()


def assert_scalar_bound(got, ref32, ref64, scale64, what):
    """A per-graph scalar of the algebra: within max(R |f32 - f64|_max, C_SUM u scale) of float64."""
    got, ref32, ref64, scale64 = map(_f64, (got, ref32, ref64, scale64))
    err = (got - ref64).abs()
    bound = torch.maximum(torch.full_like(err, R_FP32 * float((ref32 - ref64).abs().max())), C_SUM * U32 * scale64)
    i = int(torch.argmax(err - bound))
    assert bool((err <= bound).all()), (f'{what}: entry {i}: native {float(got.flatten()[i])!r}, float64 '
                                        f'{float(ref64.flatten()[i])!r}, error {float(err.flatten()[i]):.3e} > '
                                        f'{float(bound.flatten()[i]):.3e}')
    return float((err / bound.clamp(min=1e-300)).max())


# ---- the whole eval-mode forward from what its stages were fed ----------------------------------------------------------
class Restated:
    """xh0 (lig, pocket), z_t / z_0 = (lig, pocket, scale of lig), coef [n, 4], terms (Terms), out, info, gammas."""


def centred_inputs(kind, ddpm, ligand, pocket, dtype):
    """Normalised [x | h] of ligand and pocket in the frame the likelihood is evaluated in: the ligand's centre of mass
    (conditional_model.py:230-236), the pocket's ('simple', :727-735), or as given (joint; en_diffusion.py:336-360)."""
    lm, pm, n = ligand['mask'], pocket['mask'], len(ligand['size'])
    nv0, nv1, nb = ddpm.norm_values[0], ddpm.norm_values[1], ddpm.norm_biases[1]
    xl, xp = ligand['x'].to(dtype), pocket['x'].to(dtype)
    mean = lambda x, m: seg_sum(x, m, n) / seg_sum(torch.ones_like(x[:, :1]), m, n).clamp(min=1)
    if kind == 'simple':
        com = mean(xp, pm)
        xl, xp = xl - com[lm], xp - com[pm]
    xl, xp = xl / nv0, xp / nv0
    if kind == 'conditional':
        com = mean(xl, lm)
        xl, xp = xl - com[lm], xp - com[pm]
    h = lambda part: (part['one_hot'].to(dtype) - nb) / nv1
    return torch.cat([xl, h(ligand)], 1), torch.cat([xp, h(pocket)], 1)


def restate_forward(kind, ddpm, histogram, ligand, pocket, t_int, eps_t, eps_0, nets, dtype, xh0=None, z=None):
    """The eval-mode forward of ``kind`` ('conditional', 'simple', 'joint') in ``dtype`` from the raw batch, the timestep
    draw, the noise (eps = (ligand, pocket or None)) and the denoiser outputs nets = ((net_t_lig, net_t_pocket), (net_0_lig,
    net_0_pocket)).  ``xh0`` / ``z`` = (z_t, z_0) replace the restated stage inputs by what the native path fed on
    (teacher forcing); the restated ones are still returned for the stage's own comparison."""
    r = Restated()
    d = lambda x: None if x is None else x.to(dtype)
    lm, pm, n = ligand['mask'], pocket['mask'], len(ligand['size'])
    t_int = t_int.view(-1).long()
    r.xh0 = centred_inputs(kind, ddpm, ligand, pocket, dtype)
    xl, xp = r.xh0 if xh0 is None else (d(xh0[0]), d(xh0[1]))
    zero, full = torch.zeros_like(t_int), torch.full_like(t_int, ddpm.T)
    r.gamma = {k: gamma_of(ddpm, v, dtype) for k, v in (('s', t_int - 1), ('t', t_int), ('0', zero), ('T', full))}
    variant = kind
    r.z_t = noise_ref(variant, xl, d(eps_t[0]), xp, d(eps_t[1]), lm, pm, alpha_of(r.gamma['t']), sigma_of(r.gamma['t']), n, dtype)
    r.z_0 = noise_ref(variant, xl, d(eps_0[0]), xp, d(eps_0[1]), lm, pm, alpha_of(r.gamma['0']), sigma_of(r.gamma['0']), n, dtype)
    z_t, z_0 = (r.z_t, r.z_0) if z is None else ([d(v) for v in z[0]], [d(v) for v in z[1]])
    (nt_l, nt_p), (n0_l, n0_p) = nets
    r.coef = torch.stack([alpha_of(r.gamma['T']), sigma_of(r.gamma['0']) * ddpm.norm_values[1], alpha_of(r.gamma['t']),
                          sigma_of(r.gamma['t'])], 1)
    joint = kind == 'joint'
    pocket_side = (xp, eps_t[1], nt_p, z_0[1], eps_0[1], n0_p) if joint else None
    vnode = -1 if ddpm.vnode_idx is None else int(ddpm.vnode_idx)
    r.terms = vlb_terms_ref((xl, z_t[0], eps_t[0], nt_l, z_0[0], eps_0[0], n0_l), pocket_side, lm, pm, r.coef,
                            ddpm.norm_values[1], ddpm.norm_biases[1], vnode, n, dtype)
    n_lig, n_poc = ligand['size'].cpu(), pocket['size'].cpu()
    dof = {'joint': (n_lig + n_poc - 1) * 3, 'conditional': (n_lig - 1) * 3, 'simple': n_lig * 3}[kind]
    log_pn = torch.from_numpy(log_pn_numpy(histogram, n_lig.numpy(), n_poc.numpy(), conditional=not joint))
    dev = xl.device
    r.out, r.info = scalar_algebra(r.terms.terms, r.gamma['s'], r.gamma['t'], r.gamma['0'], r.gamma['T'], dof.to(dev),
                                   ddpm.norm_values[0], log_pn.to(dev), n_lig.to(dev), n_poc.to(dev), ddpm.atom_nf,
                                   ddpm.residue_nf, not joint, dtype)
    r.out['t_int'] = t_int.to(dtype)
    r.out['xh_lig_hat'] = r.terms.hat
    return r


class ForwardRecorder:
    """Keeps what each stage of one eval-mode ``forward`` received and returned: the timestep draw, the noise, and every
    denoiser call (inputs and outputs, through a forward hook on ``ddpm.dynamics``); on the native path also the calls of
    ``_native_noise`` / ``_native_noise_conditional`` and ``_native_vlb_terms``.  The wrapped methods call the originals,
    so the recorded run computes what an unrecorded one does."""

    def __init__(self, ddpm, t_inject=None):
        self.ddpm, self.t_inject = ddpm, t_inject
        self.gauss, self.combined, self.dyn, self.noise_calls, self.terms_calls = [], [], [], [], []

    def __enter__(self):
        ddpm = self.ddpm
        self._saved = {}

        def wrap(name, log):
            if not hasattr(ddpm, name):
                return
            orig = getattr(ddpm, name)
            self._saved[name] = ddpm.__dict__.get(name, None)

            def f(*a, **k):
                res = orig(*a, **k)
                log.append((a, res))
                return res
            setattr(ddpm, name, f)

        wrap('sample_gaussian', self.gauss)
        wrap('sample_combined_position_feature_noise', self.combined)
        wrap('_native_noise', self.noise_calls)
        wrap('_native_noise_conditional', self.noise_calls)
        wrap('_native_vlb_terms', self.terms_calls)
        self._hook = ddpm.dynamics.register_forward_hook(lambda m, inp, out: self.dyn.append((inp, out)))
        # the returned ``info`` dict is copied: LigandPocketDDPM.forward adds its own entries to it afterwards
        self._hook_out = ddpm.register_forward_hook(
            lambda m, inp, out: setattr(self, 'out', tuple(out[:-1]) + (dict(out[-1]),) if isinstance(out[-1], dict) else out))
        self._randint = torch.randint
        if self.t_inject is not None:
            torch.randint = lambda lo, hi, size, device=None, **k: self.t_inject.view(size).to(device)
        return self

    def __exit__(self, *exc):
        torch.randint = self._randint
        self._hook.remove()
        self._hook_out.remove()
        for name, old in self._saved.items():
            if old is None:
                self.ddpm.__dict__.pop(name, None)
            else:
                setattr(self.ddpm, name, old)

    def eps(self, kind):
        """(eps_t, eps_0), each (ligand, pocket or None), in the order forward drew them."""
        if kind == 'joint':
            (_, a), (_, b) = self.combined
            return a, b
        (_, a), (_, b) = self.gauss
        return (a, None), (b, None)

    def noisings(self):
        """The two noising calls (args, result) at t and at 0.  SimpleConditionalDDPM's goes through both wrapped methods:
        the outer call is the second of each pair."""
        return self.noise_calls if len(self.noise_calls) == 2 else self.noise_calls[1::2]

    def nets(self):
        (_, a), (_, b) = self.dyn
        return a, b
