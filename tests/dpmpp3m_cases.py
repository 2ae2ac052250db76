"""Float64 restatements of DPM-Solver++(3M) (DESIGN §15), shared by the CPU and GPU tests.

Every function takes the 3M coefficient rows the samplers use (``_fast_tables(..., 'dpmpp_3m')``: [n_graphs, 6] =
(sigma_s / sigma_t, 1 / alpha_t, sigma_t, k0, k1, k2)) and the histories m1, m2 (x0_hat of the previous step and of the one
before it), and evaluates the step in ``dtype`` on the same inputs, so that a step of either engine can be held to the
float64 value of its own fp32 inputs (``ddpm_cases.assert_fp64_bound``).  The exact closed form of the coefficient rows is
``closed_form_rows`` (mpmath)."""
import mpmath
import torch

from diffsbdd_b200.en_diffusion import scatter_mean


def _move3(z, eps, m1, m2, c, m):
    """x0_hat, z' = c0 z + k0 x0 + k1 m1 + k2 m2 (m1 not used when k1 = 0, m2 when k2 = 0), and the m2 a commit writes."""
    x0 = (z - c[m, 2:3] * eps) * c[m, 1:2]
    k1, k2 = c[m, 4:5], c[m, 5:6]
    out = c[m, 0:1] * z + c[m, 3:4] * x0 + torch.where(k1 != 0, k1 * m1, 0) + torch.where(k2 != 0, k2 * m2, 0)
    return x0, out, torch.where(k1 != 0, m1, x0)


def multistep3_ref(z, eps, m1, m2, c, pocket, lm, pm, dtype):
    """Conditional 3M step: (z', pocket', m1', m2') with the ligand COM of z' removed from all four."""
    z, eps, m1, m2, c, pocket = (x.to(dtype) for x in (z, eps, m1, m2, c, pocket))
    x0, out, sh = _move3(z, eps, m1, m2, c, lm)
    com = scatter_mean(out[:, :3], lm, dim_size=c.shape[0])
    p = pocket.clone()
    for x, m in ((out, lm), (p, pm), (x0, lm), (sh, lm)):
        x[:, :3] -= com[m]
    return out, p, x0, sh


def joint_multistep3_ref(zl, zp, eps_l, eps_p, m1l, m1p, m2l, m2p, c, lm, pm, dtype):
    """Joint 3M step: (z_lig', z_pocket', m1_lig', m1_pocket', m2_lig', m2_pocket') with the ligand + pocket COM removed."""
    zl, zp, eps_l, eps_p, m1l, m1p, m2l, m2p, c = (x.to(dtype) for x in (zl, zp, eps_l, eps_p, m1l, m1p, m2l, m2p, c))
    x0l, wl, shl = _move3(zl, eps_l, m1l, m2l, c, lm)
    x0p, wp, shp = _move3(zp, eps_p, m1p, m2p, c, pm)
    mean = scatter_mean(torch.cat((wl[:, :3], wp[:, :3])), torch.cat((lm, pm)), dim_size=c.shape[0])
    for x, m in ((wl, lm), (wp, pm), (x0l, lm), (x0p, pm), (shl, lm), (shp, pm)):
        x[:, :3] -= mean[m]
    return wl, wp, x0l, x0p, shl, shp


def cond_round3_ref(z, pocket, m1, m2, eps, noise_known, renoise, cf, cr, known, com0, fixed, lm, pm, commit, dtype):
    """Conditional RePaint round with the 3M step: the step and its COM removal, the known part noised around the pocket's
    COM, the fixed-COM alignment, the blend and the re-noise (``renoise`` None: none); every translation of the pocket moves
    both histories.  ``cr``: (alpha_s, sigma_s, alpha_{t|s}, sigma_{t|s}).  Returns (z, pocket, m1, m2)."""
    z, pocket, m1, m2, eps, cf, cr, known, com0, fixed, noise_known = (
        x.to(dtype) for x in (z, pocket, m1, m2, eps, cf, cr, known, com0, fixed, noise_known))
    n = cf.shape[0]
    x0, zu, sh = _move3(z, eps, m1, m2, cf, lm)
    m = scatter_mean(zu[:, :3], lm, dim_size=n)
    p, h1, h2 = pocket.clone(), m1.clone(), m2.clone()
    for x, mk in ((zu, lm), (p, pm), (h1, lm), (h2, lm), (x0, lm), (sh, lm)):
        x[:, :3] -= m[mk]
    xk = known.clone()
    xk[:, :3] += (scatter_mean(p[:, :3], pm, dim_size=n) - com0)[lm]
    zk = cr[lm, 0:1] * xk + cr[lm, 1:2] * noise_known
    comk = scatter_mean(zk[:, :3], lm, dim_size=n)
    zk[:, :3] -= comk[lm]
    f = fixed.bool()
    dx = scatter_mean(zu[f, :3], lm[f], dim_size=n) - scatter_mean(zk[f, :3], lm[f], dim_size=n)
    zk[:, :3] += dx[lm]
    w = fixed.view(-1, 1)
    out = zk * w + zu * (1 - w)
    move = dx - comk
    if renoise is not None:
        out = cr[lm, 2:3] * out + cr[lm, 3:4] * renoise.to(dtype)
        com2 = scatter_mean(out[:, :3], lm, dim_size=n)
        out[:, :3] -= com2[lm]
        move = move - com2
    p[:, :3] += move[pm]
    h1, h2 = (x0, sh) if commit else (h1, h2)
    h1[:, :3] += move[lm]
    h2[:, :3] += move[lm]
    return out, p, h1, h2


def _joint_noise(noise, cm, n, NL, dtype):
    nx, nhl, nhp = (x.to(dtype) for x in noise)
    ex = nx - scatter_mean(nx, cm, dim_size=n)[cm]
    return torch.cat((ex[:NL], nhl), 1), torch.cat((ex[NL:], nhp), 1)


def joint_round3_ref(zl, zp, m1l, m1p, m2l, m2p, eps_l, eps_p, noise_known, renoise, cf, cr, xl, xp, fl, fp, lm, pm, commit,
                     dtype):
    """Joint RePaint round with the 3M step; the noises are (x [NL + NP, 3], h_lig, h_pocket) as the joint kernels take them.
    The 3M COM removal and the jump back's COM removal move both histories with z.  Returns (z_lig, z_pocket, m1_lig,
    m1_pocket, m2_lig, m2_pocket)."""
    zl, zp, m1l, m1p, m2l, m2p, eps_l, eps_p, cf, cr, xl, xp, fl, fp = (
        x.to(dtype) for x in (zl, zp, m1l, m1p, m2l, m2p, eps_l, eps_p, cf, cr, xl, xp, fl, fp))
    n, NL, cm = cf.shape[0], zl.shape[0], torch.cat((lm, pm))
    x0l, ul, shl = _move3(zl, eps_l, m1l, m2l, cf, lm)
    x0p, up, shp = _move3(zp, eps_p, m1p, m2p, cf, pm)
    h = [m1l.clone(), m1p.clone(), m2l.clone(), m2p.clone()]
    m = scatter_mean(torch.cat((ul[:, :3], up[:, :3])), cm, dim_size=n)
    for x, mk in ((ul, lm), (up, pm), (x0l, lm), (x0p, pm), (shl, lm), (shp, pm), (h[0], lm), (h[1], pm), (h[2], lm), (h[3], pm)):
        x[:, :3] -= m[mk]
    el, ep = _joint_noise(noise_known, cm, n, NL, dtype)
    kl, kp = cr[lm, 0:1] * xl + cr[lm, 1:2] * el, cr[pm, 0:1] * xp + cr[pm, 1:2] * ep
    sl, sp = fl.bool(), fp.bool()
    fmask = torch.cat((lm[sl], pm[sp]))
    shift = scatter_mean(torch.cat((ul[sl, :3], up[sp, :3])), fmask, dim_size=n) - \
        scatter_mean(torch.cat((kl[sl, :3], kp[sp, :3])), fmask, dim_size=n)
    kl[:, :3] += shift[lm]
    kp[:, :3] += shift[pm]
    ol = kl * fl.view(-1, 1) + ul * (1 - fl.view(-1, 1))
    op = kp * fp.view(-1, 1) + up * (1 - fp.view(-1, 1))
    if commit:
        h = [x0l, x0p, shl, shp]
    if renoise is not None:
        el, ep = _joint_noise(renoise, cm, n, NL, dtype)
        ol, op = cr[lm, 2:3] * ol + cr[lm, 3:4] * el, cr[pm, 2:3] * op + cr[pm, 3:4] * ep
        m3 = scatter_mean(torch.cat((ol[:, :3], op[:, :3])), cm, dim_size=n)
        for x, mk in ((ol, lm), (op, pm), (h[0], lm), (h[1], pm), (h[2], lm), (h[3], pm)):
            x[:, :3] -= m3[mk]
    return (ol, op, *h)


def closed_form_rows(gamma_s, gamma_t, dps=40):
    """The exact 3M rows [N, 6] (as Python mpf) from the given gamma values, by the D1 / D2 form of DESIGN §15 with
    r0 = h1 / h, r1 = h2 / h: each k_i is the update applied to the unit vector m_i.  The last row (the first step run) is
    first order, the one before it second order (2M), the rest third order."""
    mpmath.mp.dps = dps
    gs = [mpmath.mpf(float(v)) for v in gamma_s.reshape(-1)]
    gt = [mpmath.mpf(float(v)) for v in gamma_t.reshape(-1)]
    N = len(gs)
    sig = lambda g: mpmath.sqrt(1 / (1 + mpmath.exp(-g)))
    alp = lambda g: mpmath.sqrt(1 / (1 + mpmath.exp(g)))
    hs = [(b - a) / 2 for a, b in zip(gs, gt)]
    rows = []
    for k in range(N):
        h, a_s = hs[k], alp(gs[k])
        phi1 = mpmath.exp(-h) - 1
        if k == N - 1:
            ks = [-a_s * phi1, 0, 0]
        elif k == N - 2:
            r0 = hs[k + 1] / h

            def f(m0, m1, m2):
                return -a_s * phi1 * (m0 + (m0 - m1) / (2 * r0))
            ks = [f(1, 0, 0), f(0, 1, 0), f(0, 0, 1)]
        else:
            r0, r1 = hs[k + 1] / h, hs[k + 2] / h

            def f(m0, m1, m2):
                d10, d11 = (m0 - m1) / r0, (m1 - m2) / r1
                d1 = d10 + r0 / (r0 + r1) * (d10 - d11)
                d2 = (d10 - d11) / (r0 + r1)
                return -a_s * phi1 * m0 + a_s * (phi1 / h + 1) * d1 - a_s * ((phi1 + h) / h ** 2 - mpmath.mpf(1) / 2) * d2
            ks = [f(1, 0, 0), f(0, 1, 0), f(0, 0, 1)]
        rows.append([sig(gs[k]) / sig(gt[k]), 1 / alp(gt[k]), sig(gt[k])] + [mpmath.mpf(x) for x in ks])
    return rows
