"""Float64 restatements of one RePaint round with a few-step reverse step (DESIGN §14), shared by the CPU and GPU tests.

A round takes z_t, the pocket, the 2M history and the round's draws, and returns (z, pocket, hist) of the conditional model or
(z_lig, z_pocket, hist_lig, hist_pocket) of the joint model, all evaluated in ``dtype``.  ``cf``: the step's rows of
``_fast_tables`` ([n, 3] DDIM, [n, 5] 2M); ``cr``: the RePaint rows (alpha_s, sigma_s, alpha_{t|s}, sigma_{t|s}) of
``_schedule_tables`` / ``_joint_tables``; ``noise_rev`` (DDIM at eta > 0) and ``renoise`` may be None."""
import torch

from diffsbdd_b200.en_diffusion import scatter_mean
from fast_sampler_cases import _x0_and_move


def cond_round_ref(z, pocket, hist, eps, noise_rev, noise_known, renoise, cf, cr, known, com0, fixed, lm, pm, sampler, commit,
                   dtype):
    """Conditional RePaint round: the few-step step, the known part noised around the pocket's COM, the fixed-COM alignment,
    the blend and the re-noise; every translation of the pocket moves the history too."""
    z, pocket, hist, eps, cf, cr, known, com0, fixed, noise_known = (
        x.to(dtype) for x in (z, pocket, hist, eps, cf, cr, known, com0, fixed, noise_known))
    n = cf.shape[0]
    if sampler == 'ddim':
        zu = z / cf[lm, 0:1] - cf[lm, 1:2] * eps
        if noise_rev is not None:
            zu = zu + cf[lm, 2:3] * noise_rev.to(dtype)
        x0 = hist.clone()
    else:
        x0, zu = _x0_and_move(z, eps, hist, cf, lm)
    m = scatter_mean(zu[:, :3], lm, dim_size=n)
    zu[:, :3] -= m[lm]
    p, h = pocket.clone(), hist.clone()
    p[:, :3] -= m[pm]
    h[:, :3] -= m[lm]
    x0[:, :3] -= m[lm]
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
    h = x0 if commit else h
    h[:, :3] += move[lm]
    return out, p, h


def _joint_noise(noise, cm, n, NL, dtype):
    nx, nhl, nhp = (x.to(dtype) for x in noise)
    ex = nx - scatter_mean(nx, cm, dim_size=n)[cm]
    return torch.cat((ex[:NL], nhl), 1), torch.cat((ex[NL:], nhp), 1)


def joint_round_ref(zl, zp, hl, hp, eps_l, eps_p, noise_rev, noise_known, renoise, cf, cr, xl, xp, fl, fp, lm, pm, sampler,
                    commit, dtype):
    """Joint RePaint round; the noises are (x [NL + NP, 3], h_lig, h_pocket) as the joint kernels take them.  The 2M COM
    removal and the jump back's COM removal move the history with z."""
    zl, zp, hl, hp, eps_l, eps_p, cf, cr, xl, xp, fl, fp = (
        x.to(dtype) for x in (zl, zp, hl, hp, eps_l, eps_p, cf, cr, xl, xp, fl, fp))
    n, NL, cm = cf.shape[0], zl.shape[0], torch.cat((lm, pm))
    if sampler == 'ddim':
        ul = zl / cf[lm, 0:1] - cf[lm, 1:2] * eps_l
        up = zp / cf[pm, 0:1] - cf[pm, 1:2] * eps_p
        if noise_rev is not None:
            el, ep = _joint_noise(noise_rev, cm, n, NL, dtype)
            ul, up = ul + cf[lm, 2:3] * el, up + cf[pm, 2:3] * ep
        x0l, x0p = hl.clone(), hp.clone()
    else:
        x0l, ul = _x0_and_move(zl, eps_l, hl, cf, lm)
        x0p, up = _x0_and_move(zp, eps_p, hp, cf, pm)
    hl, hp = hl.clone(), hp.clone()
    m = scatter_mean(torch.cat((ul[:, :3], up[:, :3])), cm, dim_size=n)
    for x, mk in ((ul, lm), (up, pm), (hl, lm), (hp, pm), (x0l, lm), (x0p, pm)):
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
    hl, hp = (x0l, x0p) if commit else (hl, hp)
    if renoise is not None:
        el, ep = _joint_noise(renoise, cm, n, NL, dtype)
        ol, op = cr[lm, 2:3] * ol + cr[lm, 3:4] * el, cr[pm, 2:3] * op + cr[pm, 3:4] * ep
        m3 = scatter_mean(torch.cat((ol[:, :3], op[:, :3])), cm, dim_size=n)
        for x, mk in ((ol, lm), (op, pm), (hl, lm), (hp, pm)):
            x[:, :3] -= m3[mk]
    return ol, op, hl, hp
