"""Float64 restatements of the few-step samplers of DESIGN §13 ('ddim', 'dpmpp_2m'), shared by the CPU and GPU tests.

Every function takes the coefficient rows the samplers use (``_fast_tables``: [n_graphs, 3] for DDIM, [n_graphs, 5] for 2M)
and evaluates the step's formulas in ``dtype`` on the same inputs, so that a step of either engine can be held to the float64
value of its own fp32 inputs (``ddpm_cases.assert_fp64_bound``)."""
import torch

from diffsbdd_b200.en_diffusion import scatter_mean


def ddim_ref(z, eps, noise, c, pocket, lm, pm, dtype):
    """Conditional DDIM step: z / c0 - c1 eps + c2 noise, ligand COM removed from z and the pocket (noise None: eta = 0)."""
    z, eps, c, pocket = (x.to(dtype) for x in (z, eps, c, pocket))
    out = z / c[lm, 0:1] - c[lm, 1:2] * eps
    if noise is not None:
        out = out + c[lm, 2:3] * noise.to(dtype)
    com = scatter_mean(out[:, :3], lm, dim_size=c.shape[0])
    out[:, :3] -= com[lm]
    p = pocket.clone()
    p[:, :3] -= com[pm]
    return out, p


def joint_ddim_ref(zl, zp, eps_l, eps_p, noise, c, lm, pm, dtype):
    """Joint DDIM step; ``noise`` = (x [NL + NP, 3], h_lig, h_pocket) as the joint update takes it, or None (eta = 0)."""
    zl, zp, eps_l, eps_p, c = (x.to(dtype) for x in (zl, zp, eps_l, eps_p, c))
    wl = zl / c[lm, 0:1] - c[lm, 1:2] * eps_l
    wp = zp / c[pm, 0:1] - c[pm, 1:2] * eps_p
    cm = torch.cat((lm, pm))
    if noise is not None:
        nx, nhl, nhp = (x.to(dtype) for x in noise)
        ex = nx - scatter_mean(nx, cm, dim_size=c.shape[0])[cm]
        NL = zl.shape[0]
        wl = wl + c[lm, 2:3] * torch.cat((ex[:NL], nhl), 1)
        wp = wp + c[pm, 2:3] * torch.cat((ex[NL:], nhp), 1)
    mean = scatter_mean(torch.cat((wl[:, :3], wp[:, :3])), cm, dim_size=c.shape[0])
    wl[:, :3] -= mean[lm]
    wp[:, :3] -= mean[pm]
    return wl, wp


def _x0_and_move(z, eps, hist, c, m):
    x0 = (z - c[m, 3:4] * eps) * c[m, 2:3]
    w = c[m, 4:5]
    d = torch.where(w != 0, (1 + w) * x0 - w * hist, x0)
    return x0, c[m, 0:1] * z + c[m, 1:2] * d


def multistep_ref(z, eps, hist, c, pocket, lm, pm, dtype):
    """Conditional DPM-Solver++(2M) step: (z', pocket', hist') with the ligand COM of z' removed from all three."""
    z, eps, hist, c, pocket = (x.to(dtype) for x in (z, eps, hist, c, pocket))
    x0, out = _x0_and_move(z, eps, hist, c, lm)
    com = scatter_mean(out[:, :3], lm, dim_size=c.shape[0])
    p = pocket.clone()
    out[:, :3] -= com[lm]
    p[:, :3] -= com[pm]
    x0[:, :3] -= com[lm]
    return out, p, x0


def joint_multistep_ref(zl, zp, eps_l, eps_p, hl, hp, c, lm, pm, dtype):
    """Joint DPM-Solver++(2M) step: (z_lig', z_pocket', hist_lig', hist_pocket') with the ligand + pocket COM removed."""
    zl, zp, eps_l, eps_p, hl, hp, c = (x.to(dtype) for x in (zl, zp, eps_l, eps_p, hl, hp, c))
    x0l, wl = _x0_and_move(zl, eps_l, hl, c, lm)
    x0p, wp = _x0_and_move(zp, eps_p, hp, c, pm)
    mean = scatter_mean(torch.cat((wl[:, :3], wp[:, :3])), torch.cat((lm, pm)), dim_size=c.shape[0])
    for x, m in ((wl, lm), (wp, pm), (x0l, lm), (x0p, pm)):
        x[:, :3] -= mean[m]
    return wl, wp, x0l, x0p
