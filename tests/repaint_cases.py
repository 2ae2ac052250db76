"""RePaint inpainting runs of the production graph engine recorded replay by replay, the replay schedules the eager loops
walk, and the float64 / fp32 references of the fused RePaint iterations.

Schedules.  ``conditional_schedule`` / ``joint_schedule`` / ``reverse_schedule`` list, per replay of a captured graph, its
kind, the reverse step s, the resampling round u (the conditional model's resampling index, the joint model's block
index of ``get_repaint_schedule``) and the draw purposes the replay issues, in issue order.  A joint replay followed by
the eager jump back (a frame and a jump on the same step) is marked ``eager_jump``.  ``draw_sequence`` turns a schedule
into the (draw id, role) sequence of a whole seeded run: prior, loop, partial-noising and final stages.

Recorder.  ``Recorder`` wraps, on one sampler instance, ``ConditionalDDPM._graph`` / ``EnVariationalDiffusion._joint_graph``
so that they return a proxy of the captured graph: its ``replay()`` copies the static state to the host (z, the pocket,
step, u), runs the real replay and copies what the replay wrote (t, coef3, coef4, the draw ids and every noise buffer it
filled).  It also wraps ``seeded.fill`` (the (draw id, role) of every host-side seeded draw, and the noise of the
non-loop ones) and, for the joint model, ``sample_p_zt_given_zs`` (the eager jump back between replays).  The captured
graphs themselves are the production ones; in deterministic mode a recorded call gives the same bits as an unmodified
call with the same seed.

References.  ``inpaint_update_ref`` / ``joint_inpaint_update_ref`` are the torch ops of the eager RePaint iterations
(conditional_model.py ``_inpaint``, en_diffusion.py ``_inpaint``) in a given dtype, on the fused kernels' inputs.
"""
import ctypes as C
import math
from types import SimpleNamespace

import numpy as np
import torch

import seeded_cases as sc
from diffsbdd_b200 import _native, seeded, synthetic as syn
from diffsbdd_b200.config import FULLATOM_COND, FULLATOM_JOINT
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion, scatter_mean

REV, KNOWN, RENOISE = seeded.PURPOSE_REVERSE, seeded.PURPOSE_KNOWN, seeded.PURPOSE_RENOISE
COND_ROLES = (_native.RNG_LIGAND,)
JOINT_ROLES = (_native.RNG_JOINT_X, _native.RNG_LIGAND, _native.RNG_POCKET)

N_LIG, N_POC, N_FIXED = 25, 175, 10
# the runs (T = 500): model, batch size and schedule
RUNS = {
    'inpaint_50x20': dict(joint=False, n=64, timesteps=50, resamplings=20),
    'inpaint_500x1': dict(joint=False, n=64, timesteps=500, resamplings=1),
    'joint_jump': dict(joint=True, n=16, timesteps=500, resamplings=2, jump_length=10, frames=1),
    # a frame and a jump back coincide at s = 20, 15, 10, 5, 0: the eager jump runs between replays
    'joint_frames': dict(joint=True, n=4, timesteps=25, resamplings=3, jump_length=1, frames=5),
    'diversify': dict(joint=False, n=64, noising_steps=100),
}
TORCH_SEED = 4242


def run_seeds(n):
    """One seed per sample, spread over the int63 range."""
    return [(0x9E3779B97F4A7C15 * (i + 1)) % (1 << 63) for i in range(n)]


# ---- schedules -------------------------------------------------------------------------------------------------------
def _replay(kind, s, u, purposes, eager_jump=False):
    return SimpleNamespace(kind=kind, s=s, u=u, purposes=purposes, eager_jump=eager_jump)


def conditional_schedule(timesteps, resamplings):
    """ConditionalDDPM.inpaint: per s = timesteps-1 .. 0, resamplings-1 re-noising replays and one last replay."""
    out = []
    for s in reversed(range(timesteps)):
        for u in range(resamplings):
            if u < resamplings - 1:
                out.append(_replay('inpaint_renoise', s, u, (REV, KNOWN, RENOISE)))
            else:
                out.append(_replay('inpaint_last', s, u, (REV, KNOWN)))
    return out


def reverse_schedule(first_s, n_steps):
    """Plain reverse steps s = first_s .. first_s - n_steps + 1 (sample_given_pocket, diversify)."""
    return [_replay('reverse', s, 0, (REV,)) for s in range(first_s, first_s - n_steps, -1)]


def joint_schedule(resamplings, jump_length, timesteps, return_frames=1):
    """EnVariationalDiffusion.inpaint: the blocks of get_repaint_schedule; the last step of every block but the last jumps
    back by jump_length, inside the 'inpaint_jump' replay or, when a frame is taken on that step, eagerly after an
    'inpaint' replay."""
    blocks = EnVariationalDiffusion.get_repaint_schedule(resamplings, jump_length, timesteps)
    out, s = [], timesteps - 1
    for i, n_denoise in enumerate(blocks):
        for j in range(n_denoise):
            jump = j == n_denoise - 1 and i < len(blocks) - 1
            frame = (n_denoise > jump_length or i == len(blocks) - 1) and (s * return_frames) % timesteps == 0
            if jump and not frame:
                out.append(_replay('inpaint_jump', s, i, (KNOWN, REV, RENOISE)))
            else:
                out.append(_replay('inpaint', s, i, (KNOWN, REV), eager_jump=jump))
            if jump:
                s += jump_length
            s -= 1
    return out


def schedule_of(name):
    spec = RUNS[name]
    if name == 'diversify':
        return reverse_schedule(spec['noising_steps'] - 1, spec['noising_steps'])
    if spec['joint']:
        return joint_schedule(spec['resamplings'], spec['jump_length'], spec['timesteps'], spec['frames'])
    return conditional_schedule(spec['timesteps'], spec['resamplings'])


def draw_ids(sched, first_stage=seeded.STAGE_PRIOR):
    """Draw ids of a seeded run in issue order: the first stage (prior, or partial noising for diversify), the loop
    draws of every replay (and of an eager jump after it), the final stage."""
    ids = [seeded.draw_id(first_stage)]
    for r in sched:
        ids += [seeded.draw_id(seeded.STAGE_LOOP, r.s, r.u, p) for p in r.purposes]
        if r.eager_jump:
            ids.append(seeded.draw_id(seeded.STAGE_LOOP, r.s, r.u, RENOISE))
    return ids + [seeded.draw_id(seeded.STAGE_FINAL)]


def draw_sequence(name):
    """(draw id, role) of every seeded draw of run ``name``, in issue order."""
    roles = JOINT_ROLES if RUNS[name]['joint'] else COND_ROLES
    first = seeded.STAGE_PARTIAL if name == 'diversify' else seeded.STAGE_PRIOR
    return [(i, r) for i in draw_ids(schedule_of(name), first) for r in roles]


def decode(draw):
    """(stage, s, u, purpose) of a draw id."""
    draw = int(draw)
    return draw >> 40, (draw >> 20) & 0xFFFFF, (draw >> 4) & 0xFFFF, draw & 0xF


# ---- the eager loops' coefficient ops --------------------------------------------------------------------------------
def eager_coefficients(ddpm, joint, s, timesteps, n, device, jump_length=1):
    """(t, coef3, coef4) of reverse step s as the eager loops compute them: t = (s+1)/timesteps from an s-filled tensor,
    the reverse-step coefficients of sample_p_zs_given_zt and the RePaint ones (alpha_s, sigma_s of noised_representation;
    alpha, sigma of q(z_t' | z_s) of sample_p_zt_given_zs with t' = s+1, for the joint model t' = min(s + jump, timesteps)
    as the clamped t_back column of _joint_tables)."""
    s_array = torch.full((n, 1), fill_value=s, device=device)
    t_array = (s_array + 1) / timesteps
    s_array = s_array / timesteps
    target = s_array
    gamma_s, gamma_t = ddpm.gamma(s_array), ddpm.gamma(t_array)
    if joint:
        coef3 = joint_step_coefficients(ddpm, s_array, t_array, target)
        t_back = torch.full((n, 1), fill_value=min(s + jump_length, timesteps), device=device) / timesteps
        _, sigma_j, alpha_j = ddpm.sigma_and_alpha_t_given_s(ddpm.gamma(t_back), gamma_s, target)
    else:
        coef3 = torch.cat(ddpm._step_coefficients(ddpm.gamma(s_array), ddpm.gamma(t_array), target), 1)
        _, sigma_j, alpha_j = ddpm.sigma_and_alpha_t_given_s(gamma_t, gamma_s, target)
    coef4 = torch.cat([ddpm.alpha(gamma_s, target), ddpm.sigma(gamma_s, target), alpha_j, sigma_j], 1)
    return t_array, coef3, coef4


def joint_step_coefficients(ddpm, s, t, target):
    """The coefficient ops of the eager EnVariationalDiffusion.sample_p_zs_given_zt."""
    gamma_s, gamma_t = ddpm.gamma(s), ddpm.gamma(t)
    sigma2_ts, sigma_ts, alpha_ts = ddpm.sigma_and_alpha_t_given_s(gamma_t, gamma_s, target)
    sigma_s = ddpm.sigma(gamma_s, target_tensor=target)
    sigma_t = ddpm.sigma(gamma_t, target_tensor=target)
    return torch.cat([alpha_ts, sigma2_ts / alpha_ts / sigma_t, sigma_ts * sigma_s / sigma_t], 1)


# ---- the fused RePaint kernels and their torch-op references ---------------------------------------------------------
def inpaint_update(ddpm, z, pocket, known, com0, fixed, n1, n2, coef4, lm, pm):
    """dsb_ddpm_inpaint_update on copies of (z, pocket); n2 = None: no re-noising step."""
    a, b = z.clone(), pocket.clone()
    _native.check(_native.load().dsb_ddpm_inpaint_update(
        a.data_ptr(), b.data_ptr(), known.data_ptr(), com0.data_ptr(), fixed.data_ptr(), n1.data_ptr(),
        None if n2 is None else n2.data_ptr(), coef4.data_ptr(), lm.data_ptr(), pm.data_ptr(), z.shape[0], pocket.shape[0],
        coef4.shape[0], ddpm.atom_nf, ddpm.residue_nf, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return a, b


def inpaint_update_ref(z_unknown, pocket, known, com0, fixed, n1, n2, coef, lm, pm, dtype):
    """The eager RePaint iteration of ConditionalDDPM.inpaint after the reverse step, in ``dtype`` and eager op order:
    known part following the pocket COM, noised to level s with the ligand COM removed (noised_representation), the COM
    of the fixed atoms aligned noised -> denoised, blend, and with ``n2`` the re-noising step (sample_p_zt_given_zs).
    coef = (alpha_s, sigma_s, alpha_{t|s}, sigma_{t|s}) per graph."""
    B = coef.shape[0]
    z_unknown, pocket, known, com0, fixed, n1, coef = (x.to(dtype) for x in (z_unknown, pocket, known, com0, fixed, n1, coef))
    com_pocket = scatter_mean(pocket[:, :3], pm)
    xk = known.clone()
    xk[:, :3] = known[:, :3] + (com_pocket - com0)[lm]
    zk = coef[lm, 0:1] * xk + coef[lm, 1:2] * n1
    pk = pocket.clone()
    mean = scatter_mean(zk[:, :3], lm)
    zk[:, :3] = zk[:, :3] - mean[lm]
    pk[:, :3] = pk[:, :3] - mean[pm]
    rows = fixed.bool()
    cn = scatter_mean(zk[rows][:, :3], lm[rows], dim_size=B)
    cd = scatter_mean(z_unknown[rows][:, :3], lm[rows], dim_size=B)
    dx = cd - cn
    zk[:, :3] = zk[:, :3] + dx[lm]
    pk[:, :3] = pk[:, :3] + dx[pm]
    want = zk * fixed[:, None] + z_unknown * (1 - fixed[:, None])
    if n2 is not None:
        want = coef[lm, 2:3] * want + coef[lm, 3:4] * n2.to(dtype)
        m2 = scatter_mean(want[:, :3], lm)
        want[:, :3] = want[:, :3] - m2[lm]
        pk[:, :3] = pk[:, :3] - m2[pm]
    return want, pk


def joint_noise_ref(nx, lm, pm):
    """COM-free position noise as sample_center_gravity_zero_gaussian_batch builds it from the raw draw."""
    cm = torch.cat((lm, pm))
    return nx - scatter_mean(nx, cm)[cm]


def joint_inpaint_update(ddpm, zl, zp, kn, n1, n3, coef4, lm, pm):
    """dsb_ddpm_joint_inpaint_update on copies of (zl, zp); kn = the known-part buffers (xl, xp, fl, fp); n3 = None: no
    jump back."""
    a, b = zl.clone(), zp.clone()
    P = lambda x: x.data_ptr()
    j = [None, None, None] if n3 is None else [P(x) for x in n3]
    _native.check(_native.load().dsb_ddpm_joint_inpaint_update(
        P(a), P(b), P(kn['xl']), P(kn['xp']), P(kn['fl']), P(kn['fp']), *[P(x) for x in n1], *j, P(coef4), P(lm), P(pm),
        zl.shape[0], zp.shape[0], coef4.shape[0], ddpm.atom_nf, ddpm.residue_nf, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return a, b


def joint_inpaint_update_ref(zl, zp, x0l, x0p, fl, fp, n1, n3, coef, lm, pm, dtype):
    """The eager RePaint iteration of EnVariationalDiffusion.inpaint around the reverse step, in ``dtype``: (zl, zp) = the
    denoised sample; known part alpha_s x0 + sigma_s eps1, shifted so that the COM of the fixed ligand+pocket nodes
    matches the denoised one, blend, and with ``n3`` the jump back (sample_p_zt_given_zs, joint COM removed).  n1, n3 =
    raw (nx [NL+NP, 3], nh_lig, nh_pocket) draws."""
    B, NL = coef.shape[0], zl.shape[0]
    cm = torch.cat((lm, pm))
    zl, zp, x0l, x0p, fl, fp, coef = (x.to(dtype) for x in (zl, zp, x0l, x0p, fl, fp, coef))
    nx, nhl, nhp = (x.to(dtype) for x in n1)
    ex = joint_noise_ref(nx, lm, pm)
    zkl = coef[lm, 0:1] * x0l + coef[lm, 1:2] * torch.cat((ex[:NL], nhl), 1)
    zkp = coef[pm, 0:1] * x0p + coef[pm, 1:2] * torch.cat((ex[NL:], nhp), 1)
    sel_l, sel_p = fl.bool(), fp.bool()
    idx = torch.cat((lm[sel_l], pm[sel_p]))
    com_u = scatter_mean(torch.cat((zl[sel_l][:, :3], zp[sel_p][:, :3])), idx, dim_size=B)
    com_k = scatter_mean(torch.cat((zkl[sel_l][:, :3], zkp[sel_p][:, :3])), idx, dim_size=B)
    shift = com_u - com_k
    zkl[:, :3] += shift[lm]
    zkp[:, :3] += shift[pm]
    wl = zkl * fl[:, None] + zl * (1 - fl[:, None])
    wp = zkp * fp[:, None] + zp * (1 - fp[:, None])
    if n3 is not None:
        n3x, n3l, n3p = (x.to(dtype) for x in n3)
        e3 = joint_noise_ref(n3x, lm, pm)
        wl = coef[lm, 2:3] * wl + coef[lm, 3:4] * torch.cat((e3[:NL], n3l), 1)
        wp = coef[pm, 2:3] * wp + coef[pm, 3:4] * torch.cat((e3[NL:], n3p), 1)
        mean = scatter_mean(torch.cat((wl[:, :3], wp[:, :3])), cm)
        wl[:, :3] -= mean[lm]
        wp[:, :3] -= mean[pm]
    return wl, wp


def joint_jump_ref(ddpm, zl, zp, eps_l, eps_p, gamma_t, gamma_s, lm, pm, dtype):
    """The eager jump back (sample_p_zt_given_zs) on its recorded input and noise (eps.x already COM-free), in ``dtype``."""
    zl, zp, eps_l, eps_p, gamma_t, gamma_s = (x.to(dtype) for x in (zl, zp, eps_l, eps_p, gamma_t, gamma_s))
    _, sigma, alpha = ddpm.sigma_and_alpha_t_given_s(gamma_t, gamma_s, zl)
    wl, wp = alpha[lm] * zl + sigma[lm] * eps_l, alpha[pm] * zp + sigma[pm] * eps_p
    mean = scatter_mean(torch.cat((wl[:, :3], wp[:, :3])), torch.cat((lm, pm)))
    wl[:, :3] -= mean[lm]
    wp[:, :3] -= mean[pm]
    return wl, wp


# ---- inputs ----------------------------------------------------------------------------------------------------------
def fixed_first(n_graphs, n_lig=N_LIG, n_fixed=N_FIXED):
    """0/1 per ligand row: the first n_fixed atoms of every graph known (bench.py inpaint_inputs layout)."""
    f = torch.zeros(n_graphs * n_lig)
    f.view(n_graphs, n_lig)[:, :n_fixed] = 1
    return f


def complex_inputs(joint, n_graphs, seed=3):
    """Ligand and pocket dicts of n_graphs synthetic complexes of 25 + 175 atoms (ligands around the pocket COM), the
    ligand fixed mask and, for the joint model, the pocket fixed mask (every third pocket node free)."""
    cfg = FULLATOM_JOINT if joint else FULLATOM_COND
    d = syn.synthetic_complex_batch(cfg, [N_LIG] * n_graphs, [N_POC] * n_graphs, seed=seed)
    lig = {'x': d['lig_coords'], 'one_hot': d['lig_one_hot'], 'size': d['num_lig_atoms'], 'mask': d['lig_mask']}
    pocket = {'x': d['pocket_coords'], 'one_hot': d['pocket_one_hot'], 'size': d['num_pocket_nodes'], 'mask': d['pocket_mask']}
    pfix = torch.ones(n_graphs * N_POC)
    pfix[::3] = 0
    to = lambda dct: {k: v.cuda() for k, v in dct.items()}
    return to(lig), to(pocket), fixed_first(n_graphs).cuda(), pfix.cuda()


def call(ddpm, name, seeds=None):
    """One sampler call of run ``name`` (fresh input dicts: the samplers normalise them in place).  diversify is called
    right after a sample_given_pocket call on the same sampler, as its own part of the call."""
    spec = RUNS[name]
    lig, pocket, fixed, pfix = complex_inputs(spec['joint'], spec['n'])
    torch.manual_seed(TORCH_SEED)
    if name == 'diversify':
        return ddpm.diversify(lig, pocket, spec['noising_steps'], seeds=seeds)
    if spec['joint']:
        return ddpm.inpaint(lig, pocket, fixed, pfix, resamplings=spec['resamplings'], jump_length=spec['jump_length'],
                            return_frames=spec['frames'], timesteps=spec['timesteps'], seeds=seeds)
    return ddpm.inpaint(lig, pocket, fixed, resamplings=spec['resamplings'], timesteps=spec['timesteps'], center='ligand',
                        seeds=seeds)


def sample_before_diversify(ddpm, seeds=None):
    """The sample_given_pocket call (configs[2] batch, 500 steps) whose captured 'reverse' graph diversify replays."""
    _, pocket, _, _ = complex_inputs(False, RUNS['diversify']['n'])
    torch.manual_seed(TORCH_SEED + 1)
    return ddpm.sample_given_pocket(pocket, torch.full((RUNS['diversify']['n'],), N_LIG, device='cuda'), seeds=seeds)


# ---- recorder --------------------------------------------------------------------------------------------------------
class _RecordingGraph:
    """Stands in for a captured graph: replay() records the static state around the real replay."""

    def __init__(self, rec, st, kind, graph):
        self.rec, self.st, self.kind, self.graph = rec, st, kind, graph

    def replay(self):
        rec, st, kind = self.rec, self.st, self.kind
        zk, pk = ('zl', 'zp') if rec.joint else ('z', 'pocket')
        if rec.ctx is None:
            rec.ctx = _context(st, rec.joint)
        r = dict(kind=kind, graph=self.graph, step=int(st['step']), u=int(st['u']) if st['seeded'] else None,
                 z=st[zk].cpu(), p=st[pk].cpu() if rec.joint else st[pk][:, :3].cpu())
        self.graph.replay()
        r.update(t=st['t'].cpu(), coef3=st['coef3'].cpu(), coef4=st['coef4'].cpu(), out_z=st[zk].cpu(),
                 out_p=st[pk].cpu() if rec.joint else st[pk][:, :3].cpu())
        if rec.joint:
            r['n_rev'] = tuple(x.cpu() for x in st['n_rev'])
            if kind != 'reverse':
                r['n_known'] = tuple(x.cpu() for x in st['n_known'])
            if kind == 'inpaint_jump':
                r['n_jump'] = tuple(x.cpu() for x in st['n_jump'])
        else:
            r['noise'] = st['noise'].cpu()
            if kind != 'reverse':
                r['noise1'] = st['noise1'].cpu()
            if kind == 'inpaint_renoise':
                r['noise2'] = st['noise2'].cpu()
            r['h_same'] = torch.equal(st['pocket'][:, 3:], rec.ctx['h0'])
        if st['seeded']:
            r['draw'] = st['draw'].cpu()
            order = {'reverse': (REV,), 'inpaint_last': (REV, KNOWN), 'inpaint_renoise': (REV, KNOWN, RENOISE),
                     'inpaint': (KNOWN, REV), 'inpaint_jump': (KNOWN, REV, RENOISE)}[kind]
            roles = JOINT_ROLES if rec.joint else COND_ROLES
            rec.draws += [(int(r['draw'][p]), role) for p in order for role in roles]
        rec.replays.append(r)


def _context(st, joint):
    """The static buffers a run's replays read but never write (kept on the device)."""
    ctx = dict(lm=st['lig_mask'].clone(), pm=st['pocket_mask'].clone(), seeds=st['seeds'].clone() if st['seeded'] else None)
    if joint:
        if st['known'] is not None:
            ctx['known'] = {k: v.clone() for k, v in st['known'].items()}
    else:
        ctx['h0'] = st['pocket'][:, 3:].clone()
        if st['inpaint'] is not None:
            ctx['inpaint'] = {k: v.clone() for k, v in st['inpaint'].items()}
    return ctx


class Recorder:
    """Context manager recording one (or more) sampler calls on ``ddpm``: ``replays`` (one dict per graph replay),
    ``jumps`` (index of the replay an eager jump followed -> its input, noise and output), ``draws`` ((draw id, role)
    of every seeded draw, in issue order), ``fills`` (draw id -> {role: noise} of the host-side seeded draws outside the
    loop: prior, partial noising, final, eager jumps) and ``partial`` (diversify's partially_noised_ligand input and
    output).  Works for either engine: the eager one only adds ``draws`` and ``fills``."""

    def __init__(self, ddpm, joint):
        self.ddpm, self.joint = ddpm, joint
        self.replays, self.jumps, self.draws, self.fills, self.partial = [], {}, [], {}, None
        self.ctx, self._building, self._in_jump = None, 0, False

    def __enter__(self):
        d, rec = self.ddpm, self
        name = '_joint_graph' if self.joint else '_graph'
        orig_graph = getattr(d, name)

        def graph(st, kind, *args):
            rec._building += 1                  # capture and warm-up: their seeded.fill calls are not draws of the run
            try:
                g = orig_graph(st, kind, *args)
            finally:
                rec._building -= 1
            return _RecordingGraph(rec, st, kind, g)
        setattr(d, name, graph)

        self._orig_fill = orig_fill = seeded.fill

        def fill(out, role, seeds, draw, lig_mask, pocket_mask, kind=_native.RNG_NORMAL):
            res = orig_fill(out, role, seeds, draw, lig_mask, pocket_mask, kind)
            if not rec._building:
                i = int(draw[0])
                rec.draws.append((i, role))
                if decode(i)[0] != seeded.STAGE_LOOP or rec._in_jump:
                    rec.fills.setdefault(i, {})[role] = out.cpu()
            return res
        seeded.fill = fill

        if self.joint:
            orig_zt = d.sample_p_zt_given_zs

            def zt(zl, zp, lm, pm, gamma_t, gamma_s, fix_noise=False):
                if not d._joint_use_graph(zl.device):
                    return orig_zt(zl, zp, lm, pm, gamma_t, gamma_s, fix_noise)
                noise = []
                orig_noise = d.sample_combined_position_feature_noise

                def capture(li, pi):
                    noise.append(orig_noise(li, pi))
                    return noise[-1]
                inp = dict(zl=zl.cpu(), zp=zp.cpu(), gamma_t=gamma_t.cpu(), gamma_s=gamma_s.cpu())
                d.sample_combined_position_feature_noise, rec._in_jump = capture, True
                try:
                    out = orig_zt(zl, zp, lm, pm, gamma_t, gamma_s, fix_noise)
                finally:
                    del d.sample_combined_position_feature_noise
                    rec._in_jump = False
                inp.update(eps=tuple(x.cpu() for x in noise[0]), out=tuple(x.cpu() for x in out))
                rec.jumps[len(rec.replays) - 1] = inp
                return out
            d.sample_p_zt_given_zs = zt
        else:
            orig_partial = d.partially_noised_ligand

            def partial(ligand, pocket, noising_steps):
                inp = dict(x=ligand['x'].clone(), one_hot=ligand['one_hot'].clone(), px=pocket['x'].clone(),
                           ph=pocket['one_hot'].clone(), lm=ligand['mask'].clone(), pm=pocket['mask'].clone(),
                           noising_steps=noising_steps)
                out = orig_partial(ligand, pocket, noising_steps)
                rec.partial = dict(inp=inp, out=tuple(x.clone() for x in out))
                return out
            d.partially_noised_ligand = partial
        return self

    def __exit__(self, *exc):
        d = self.ddpm
        del d.__dict__['_joint_graph' if self.joint else '_graph']
        seeded.fill = self._orig_fill
        if self.joint:
            del d.sample_p_zt_given_zs
        else:
            del d.partially_noised_ligand
        return False


# ---- comparisons -----------------------------------------------------------------------------------------------------
def ulp_of(x):
    return 2.0 ** (math.floor(math.log2(x)) - 23) if x > 0 else 0.0


def assert_restated(got, role, cols, seeds, draw, lm, pm, what):
    """``got`` (host fp32 [rows, cols]) is the seeded normal draw ``draw`` of ``role``: within 8 ulp of max(|z|, 1) of the
    numpy restatement (seeded_cases), the contract of the seeded generator."""
    want = sc.normals(sc.words(role, cols, seeds, draw, lm, pm))[:, :cols]
    g = got.numpy().astype(np.float64)
    assert g.shape == want.shape, (what, g.shape, want.shape)
    err = np.abs(g - want)
    assert np.all(err <= 8 * 2.0 ** -23 * np.maximum(np.abs(want), 1.0)), f'{what}: max |err| {float(err.max()):.3e}'
