"""Sampling-side members of the reference's ``ConditionalDDPM`` (pocket-conditioned ligand DDPM).

reference: equivariant_diffusion/conditional_model.py — ``sample_given_pocket`` (:479-555), ``inpaint``
(:558-686), ``diversify`` (:364-409), ``sample_p_zs_given_zt`` (:432-464), ``sample_p_xh_given_z0`` (:112-135),
``sample_normal_zero_com`` (:140-160), ``noised_representation`` (:162-183), ``sample_p_zt_given_zs``
(:420-430), ``remove_mean_batch`` (:688-696), ``SimpleConditionalDDPM`` (:702-746), and the eval-mode likelihood ``forward``
(:202-330, :727-735) with ``kl_prior``, ``log_pxh_given_z0_without_constants`` and ``log_pN`` (training is not built).

Two loop engines produce the same distribution:

* eager  — the reference's own Python loop, step by step (same torch ops and RNG call order; used for
  trajectory parity tests and whenever the denoiser is not the native CUDA module);
* graph  — SURVEY.md §8(f1): one reverse step (schedule lookup -> native denoiser -> randn -> fused
  mu/sigma update + COM removal, libdiffsbdd_b200 ``dsb_ddpm_ligand_update``) is captured ONCE as a CUDA
  graph and replayed ``timesteps`` times; the reference's per-step host syncs (mean-zero assert, NaN
  check) become sticky device flags / a final check.  Selected automatically on CUDA with the native
  denoiser; ``ddpm.loop_engine = 'eager'`` forces the reference-order loop.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn.functional as F

from . import _native, seeded
from .dynamics import EGNNDynamics
from .en_diffusion import (MULTISTEP, EnVariationalDiffusion, check_sampler, follows_dynamics_determinism, multistep_update,
                           scatter_add, scatter_mean, num_nodes_to_batch_mask)


class ConditionalDDPM(EnVariationalDiffusion):
    """reference conditional_model.py:12."""

    loop_engine = 'auto'   # 'auto' | 'graph' | 'eager'

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        assert not self.dynamics.update_pocket_coords      # conditional_model.py:18
        self._graph_cache = {}

    # ---- elementary sampling steps ---------------------------------------------------------------------
    @classmethod
    def remove_mean_batch(cls, x_lig, x_pocket, lig_indices, pocket_indices):
        """conditional_model.py:688-696: subtract the LIGAND centre of mass from ligand and pocket."""
        mean = scatter_mean(x_lig, lig_indices, dim=0)
        return x_lig - mean[lig_indices], x_pocket - mean[pocket_indices]

    def sample_normal(self, *args):
        raise NotImplementedError("Has been replaced by sample_normal_zero_com()")

    def sample_normal_zero_com(self, mu_lig, xh0_pocket, sigma, lig_mask, pocket_mask, fix_noise=False):
        """conditional_model.py:140-160."""
        if fix_noise:
            raise NotImplementedError("fix_noise option isn't implemented yet")
        eps = self._lig_noise(lig_mask, self.n_dims + self.atom_nf)
        out_lig = mu_lig + sigma[lig_mask] * eps
        xh_pocket = xh0_pocket.detach().clone()
        out_lig[:, :self.n_dims], xh_pocket[:, :self.n_dims] = self.remove_mean_batch(
            out_lig[:, :self.n_dims], xh0_pocket[:, :self.n_dims], lig_mask, pocket_mask)
        return out_lig, xh_pocket

    def noised_representation(self, xh_lig, xh0_pocket, lig_mask, pocket_mask, gamma_t):
        """conditional_model.py:162-183: z_t ~ q(z_t | x, h) for the ligand; pocket follows the COM shift."""
        alpha_t, sigma_t = self.alpha(gamma_t, xh_lig), self.sigma(gamma_t, xh_lig)
        eps = self._lig_noise(lig_mask, self.n_dims + self.atom_nf)
        z_lig = alpha_t[lig_mask] * xh_lig + sigma_t[lig_mask] * eps
        xh_pocket = xh0_pocket.detach().clone()
        z_lig[:, :self.n_dims], xh_pocket[:, :self.n_dims] = self.remove_mean_batch(
            z_lig[:, :self.n_dims], xh_pocket[:, :self.n_dims], lig_mask, pocket_mask)
        return z_lig, xh_pocket, eps

    def sample_p_zt_given_zs(self, zs_lig, xh0_pocket, ligand_mask, pocket_mask, gamma_t, gamma_s, fix_noise=False):
        """conditional_model.py:420-430: forward (re-noising) step of RePaint."""
        _, sigma_ts, alpha_ts = self.sigma_and_alpha_t_given_s(gamma_t, gamma_s, zs_lig)
        return self.sample_normal_zero_com(alpha_ts[ligand_mask] * zs_lig, xh0_pocket, sigma_ts, ligand_mask,
                                           pocket_mask, fix_noise)

    def _step_coefficients(self, gamma_s, gamma_t, target):
        """(alpha_{t|s}, sigma^2_{t|s}/alpha_{t|s}/sigma_t, sigma_{t|s} sigma_s / sigma_t) — conditional_model.py:435-456."""
        sigma2_ts, sigma_ts, alpha_ts = self.sigma_and_alpha_t_given_s(gamma_t, gamma_s, target)
        sigma_s = self.sigma(gamma_s, target_tensor=target)
        sigma_t = self.sigma(gamma_t, target_tensor=target)
        return alpha_ts, sigma2_ts / alpha_ts / sigma_t, sigma_ts * sigma_s / sigma_t

    def sample_p_zs_given_zt(self, s, t, zt_lig, xh0_pocket, ligand_mask, pocket_mask, fix_noise=False):
        """conditional_model.py:432-464: one reverse step z_t -> z_s (eager, reference op order)."""
        alpha_ts, coef_eps, sigma = self._step_coefficients(self.gamma(s), self.gamma(t), zt_lig)
        eps_lig, _ = self.dynamics(zt_lig, xh0_pocket, t, ligand_mask, pocket_mask)
        mu_lig = zt_lig / alpha_ts[ligand_mask] - coef_eps[ligand_mask] * eps_lig
        zs_lig, xh0_pocket = self.sample_normal_zero_com(mu_lig, xh0_pocket, sigma, ligand_mask, pocket_mask, fix_noise)
        self.assert_mean_zero_with_mask(zt_lig[:, :self.n_dims], ligand_mask)
        return zs_lig, xh0_pocket

    def sample_p_xh_given_z0(self, z0_lig, xh0_pocket, lig_mask, pocket_mask, batch_size, fix_noise=False):
        """conditional_model.py:112-135: final x ~ p(x | z_0), argmax atom types."""
        t_zeros = torch.zeros(size=(batch_size, 1), device=z0_lig.device)
        gamma_0 = self.gamma(t_zeros)
        sigma_x = self.SNR(-0.5 * gamma_0)
        net_out, _ = self.dynamics(z0_lig, xh0_pocket, t_zeros, lig_mask, pocket_mask)
        mu_x = self.compute_x_pred(net_out, z0_lig, gamma_0, lig_mask)
        xh_lig, xh0_pocket = self.sample_normal_zero_com(mu_x, xh0_pocket, sigma_x, lig_mask, pocket_mask, fix_noise)
        x_lig, h_lig = self.unnormalize(xh_lig[:, :self.n_dims], z0_lig[:, self.n_dims:])
        x_pocket, h_pocket = self.unnormalize(xh0_pocket[:, :self.n_dims], xh0_pocket[:, self.n_dims:])
        h_lig = F.one_hot(torch.argmax(h_lig, dim=1), self.atom_nf)
        return x_lig, h_lig, x_pocket, h_pocket

    def sample_combined_position_feature_noise(self, lig_indices, xh0_pocket, pocket_indices):
        raise NotImplementedError("Use sample_normal_zero_com() instead.")

    def sample(self, *args):
        raise NotImplementedError("Conditional model does not support sampling without given pocket.")

    # ---- CUDA-graphed reverse loop (SURVEY.md §8 f1, f2) ------------------------------------------------
    def _use_graph(self, device) -> bool:
        if self.loop_engine == 'eager':
            return False
        ok = isinstance(self.dynamics, EGNNDynamics) and torch.device(device).type == 'cuda'
        if self.loop_engine == 'graph' and not ok:
            raise RuntimeError("loop_engine='graph' needs the native EGNNDynamics on a CUDA device")
        return ok

    def _schedule_tables(self, steps, timesteps, device):
        """Per-step scalars for s = 0..steps-1 (t = s+1), computed with the same fp32 torch ops as the
        eager step so both engines use bit-identical coefficients.  Columns of the second table:
        reverse step (alpha_{t|s}, sigma^2_{t|s}/alpha_{t|s}/sigma_t, sigma_{t|s} sigma_s/sigma_t) |
        inpainting (alpha_s, sigma_s, alpha_{t|s}, sigma_{t|s}) — conditional_model.py:162-183, :420-430."""
        s_int = torch.arange(steps, device=device).view(-1, 1)
        t_arr = (s_int + 1) / timesteps
        s_arr = s_int / timesteps
        gamma_s, gamma_t = self.gamma(s_arr), self.gamma(t_arr)
        a, c, sg = self._step_coefficients(gamma_s, gamma_t, s_arr)
        _, sigma_ts, alpha_ts = self.sigma_and_alpha_t_given_s(gamma_t, gamma_s, s_arr)
        inp = [self.alpha(gamma_s, s_arr), self.sigma(gamma_s, s_arr), alpha_ts, sigma_ts]
        return t_arr.float().contiguous(), torch.cat([a, c, sg] + inp, dim=1).float().contiguous()

    def _engine(self, z_lig, xh_pocket, lig_mask, pocket_mask, n_samples, timesteps, seeds=None, sampler='ddpm', eta=0.0,
                top=None):
        """Static buffers + captured graphs for one batch layout.  A cached engine is reused only while everything a
        captured graph bakes in is unchanged: batch layout (mask contents), the native module generation (packed-weight
        blob), its arithmetic mode and its workspace/status buffers, whether its noise is seeded (the seeds themselves
        are a static buffer, refreshed on every call), the sampler with its eta, and the top of its grid (``top``: as
        _fast_tables; diversify's t*)."""
        device = z_lig.device
        dyn: EGNNDynamics = self.dynamics
        dyn._ensure_handle(device)
        key = (tuple(z_lig.shape), tuple(xh_pocket.shape), n_samples, timesteps, str(device), seeds is not None, sampler, eta)
        if top is not None:
            key += (top,)
        st = self._graph_cache.get(key)
        if st is not None:
            same_layout = torch.equal(st['lig_mask'], lig_mask) and torch.equal(st['pocket_mask'], pocket_mask)
            if not same_layout or st['sig'] != dyn.capture_signature():
                st = None            # re-capture: a replay would use stale masks / freed weights / another kernel selection
        if st is None:
            self._graph_cache.clear()
            t_table, coef_table = self._schedule_tables(timesteps, timesteps, device)
            # the captured steps own static copies of the masks, so one capture serves every later batch with the
            # same layout (generate_ligands builds fresh mask tensors on every call)
            st = dict(
                z=torch.empty_like(z_lig), pocket=torch.empty_like(xh_pocket), noise=torch.empty_like(z_lig),
                noise1=torch.empty_like(z_lig), noise2=torch.empty_like(z_lig),
                t=torch.zeros((n_samples, 1), device=device), coef3=torch.zeros((n_samples, 3), device=device),
                coef4=torch.zeros((n_samples, 4), device=device),
                step=torch.zeros(1, dtype=torch.int64, device=device), t_table=t_table, coef_table=coef_table,
                lig_mask=lig_mask.clone(), pocket_mask=pocket_mask.clone(), graphs={}, sig=None,
                n_samples=n_samples, inpaint=None, seeded=seeds is not None)
            if seeds is not None:     # seeds, draw ids of the step's three draws, resampling round u
                st.update(seeds=torch.empty_like(seeds), draw=torch.zeros(3, dtype=torch.int64, device=device),
                          u=torch.zeros(1, dtype=torch.int64, device=device))
            if sampler != 'ddpm':     # few-step samplers: their coefficient table; DDIM at eta = 0 adds 0 * (zeroed noise)
                fast_t, fast = self._fast_tables(timesteps, sampler, eta, device, top)
                st.update(fast_t=fast_t, fast_table=fast, coef_fast=torch.zeros((n_samples, fast.shape[1]), device=device),
                          eta=eta, sampler=sampler)
                st['noise'].zero_()
                if sampler in MULTISTEP:   # RePaint rounds: the 2M / 3M row and the RePaint row in one [n, 9 | 10] buffer
                    st['hist'] = torch.zeros_like(z_lig)
                    if sampler == 'dpmpp_3m':
                        st['hist2'] = torch.zeros_like(z_lig)
                    ms = torch.cat((fast, coef_table[:, 3:]), 1).contiguous()
                    st['ms_table'] = ms
                    st['coef9' if sampler == 'dpmpp_2m' else 'coef10'] = torch.zeros((n_samples, ms.shape[1]), device=device)
            self._graph_cache[key] = st
        if seeds is not None:
            st['seeds'].copy_(seeds)
            st['u'].zero_()
        return st

    def _captured_step(self, st, kind):
        """One iteration as a python callable over the static buffers of ``st``, with the step of the sampler the engine was
        built for.  kind: 'reverse' ('ddpm') | 'ddim' | 'dpmpp_2m' | 'dpmpp_3m' (z_t -> z_s, step -= 1) | 'inpaint_renoise'
        (the step + RePaint blend + re-noise to t, u += 1; 2M / 3M: the round does not commit) | 'inpaint_last' (the step +
        blend, step -= 1, u = 0; 2M / 3M: the last round of the step commits its x0_hat as the history) (DESIGN §13-15).
        A run: draw ids -> the step's table rows -> native denoiser -> draws -> dsb_ddpm_ligand_update (+
        dsb_ddpm_inpaint_update), or the 2M / 3M step or RePaint round (_native.multistep_update) -> counters."""
        dyn: EGNNDynamics = self.dynamics
        lib = _native.load()
        lm, pm, n = st['lig_mask'], st['pocket_mask'], st['n_samples']
        sizes = (st['z'].shape[0], st['pocket'].shape[0], n, self.atom_nf, self.residue_nf)
        ptr = lambda x: None if x is None else x.data_ptr()
        sampler = st.get('sampler', 'ddpm')
        repaint, renoise = kind.startswith('inpaint'), kind == 'inpaint_renoise'
        # table rows -> the buffers the kernels read, {table: [(buffer, first column)]}; one index_select per table
        coef = 'coef3' if sampler == 'ddpm' else 'coef_fast'
        if repaint and sampler in MULTISTEP:      # the 2M / 3M row and the RePaint row in one [n, 9 | 10] buffer
            coef = 'coef9' if sampler == 'dpmpp_2m' else 'coef10'
            stage = {'ms_table': [(coef, 0)]}
        else:
            stage = {'coef_table' if sampler == 'ddpm' else 'fast_table': [(coef, 0)]}
            if repaint:                           # the RePaint row of dsb_ddpm_inpaint_update
                stage.setdefault('coef_table', []).append(('coef4', 3))
        t_table = 't_table' if sampler == 'ddpm' else 'fast_t'     # fast_t: diversify's top moves the few-step grid
        # the step's draws in eager order: reverse noise ('ddpm', DDIM at eta > 0), known part, re-noise
        draws = [(p, buf) for p, buf, on in ((seeded.PURPOSE_REVERSE, 'noise', sampler == 'ddpm' or st.get('eta', 0) > 0),
                                             (seeded.PURPOSE_KNOWN, 'noise1', repaint),
                                             (seeded.PURPOSE_RENOISE, 'noise2', renoise)) if on]

        def run():
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            if st['seeded'] and draws:
                seeded.graph_draw_ids(st['step'], st['u'], st['draw'])
            idx = st['step'].clamp(min=0)
            st['t'].copy_(st[t_table].index_select(0, idx).expand(n, 1))
            for table, bufs in stage.items():
                row = st[table].index_select(0, idx)
                for key, c0 in bufs:
                    st[key].copy_(row[:, c0:c0 + st[key].shape[1]].expand_as(st[key]))
            eps, _ = dyn(st['z'], st['pocket'], st['t'], lm, pm)
            for p, buf in draws:
                if st['seeded']:
                    seeded.fill(st[buf], _native.RNG_LIGAND, st['seeds'], st['draw'][p:p + 1], lm, pm)
                else:
                    st[buf].normal_()
            ip = st['inpaint']
            n2 = st['noise2'] if renoise else None
            if sampler in MULTISTEP:
                rp = ((ip['known'], None, ip['com0'], ip['fixed'], None, st['noise1'], None, None, n2, None, None) if repaint
                      else ())
                _native.multistep_update(lib, (st['z'], st['pocket']), self._static_history(st), (eps, None), st[coef],
                                         (lm, pm), sizes, 0, stream, rp, int(not renoise))
            else:
                _native.check(lib.dsb_ddpm_ligand_update(
                    ptr(st['z']), ptr(eps), ptr(st['noise']), ptr(st[coef]), ptr(lm), ptr(pm), ptr(st['pocket']), *sizes,
                    ptr(st['z']), ptr(st['pocket']), stream))
                if repaint:
                    _native.check(lib.dsb_ddpm_inpaint_update(
                        ptr(st['z']), ptr(st['pocket']), ptr(ip['known']), ptr(ip['com0']), ptr(ip['fixed']), ptr(st['noise1']),
                        ptr(n2), ptr(st['coef4']), ptr(lm), ptr(pm), *sizes, stream))
            if renoise:
                if st['seeded']:
                    st['u'].add_(1)
            else:
                st['step'].sub_(1)
                if st['seeded'] and kind == 'inpaint_last':
                    st['u'].zero_()
        return run

    @staticmethod
    def _start(st, z_lig, xh_pocket, first_s):
        """Loads the static state a run of captured steps starts from: z, pocket, step and (seeded) the resampling round
        u = 0.  A warm-up run advances u like any other, so capture resets it here as well."""
        st['z'].copy_(z_lig); st['pocket'].copy_(xh_pocket); st['step'].fill_(first_s)
        if st['seeded']:
            st['u'].zero_()
        for key in ('hist', 'hist2'):
            if key in st:
                st[key].zero_()

    @staticmethod
    def _static_history(st):
        """The multistep histories of the static state, newest first, as (ligand, no pocket part) pairs."""
        return tuple((st[k], None) for k in ('hist', 'hist2') if k in st)

    def _graph(self, st, kind, z_lig, xh_pocket, first_s):
        """Captured CUDA graph of ``kind`` (captured on first use; capture leaves the static state as it found it)."""
        g = st['graphs'].get(kind)
        if g is not None:
            return g
        device = z_lig.device
        dyn: EGNNDynamics = self.dynamics
        run = self._captured_step(st, kind)

        def reset():
            self._start(st, z_lig, xh_pocket, first_s)

        # warm-up on a side stream (allocator + plan caches + workspace), restoring RNG and state afterwards.  It runs on the
        # real inputs: the static buffers start uninitialised, and a NaN left there by an earlier allocation would set the
        # sticky NaN flag that the deferred status check reports after the loop.
        rng = torch.cuda.get_rng_state(device)
        reset()
        side = torch.cuda.Stream(device=device)
        side.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(side):
            run()
        torch.cuda.current_stream(device).wait_stream(side)
        torch.cuda.set_rng_state(rng, device)
        reset()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            run()
        reset()
        st['graphs'][kind] = g
        sig = dyn.capture_signature()
        if st['sig'] is not None and st['sig'] != sig:      # e.g. the workspace grew during this warm-up: older captures are stale
            st['graphs'] = {kind: g}
        st['sig'] = sig
        return g

    def _graphed_reverse_steps(self, z_lig, xh_pocket, lig_mask, pocket_mask, n_samples, first_s, n_steps, timesteps):
        """Runs reverse steps s = first_s, first_s-1, ..., first_s-n_steps+1 by replaying one captured step."""
        dyn: EGNNDynamics = self.dynamics
        st = self._engine(z_lig, xh_pocket, lig_mask, pocket_mask, n_samples, timesteps, self._seeds())
        prev_defer = dyn.defer_status_check
        dyn.defer_status_check = True
        try:
            g = self._graph(st, 'reverse', z_lig, xh_pocket, first_s)
            self._start(st, z_lig, xh_pocket, first_s)
            for _ in range(n_steps):
                g.replay()
        finally:
            dyn.defer_status_check = prev_defer
        dyn.check_status()
        return st['z'].clone(), st['pocket'].clone()

    def _graphed_fast_loop(self, z_lig, xh_pocket, lig_mask, pocket_mask, n_samples, timesteps, sampler, eta, return_frames,
                           out_lig, out_pocket, top=None):
        """The whole 'ddim' / 'dpmpp_2m' / 'dpmpp_3m' reverse loop as ``timesteps`` replays of one captured step; frames are
        copied from the static state between replays, so the history of the multistep samplers runs through them.  ``top``:
        the grid's top t as _fast_tables takes it (diversify)."""
        dyn: EGNNDynamics = self.dynamics
        st = self._engine(z_lig, xh_pocket, lig_mask, pocket_mask, n_samples, timesteps, self._seeds(), sampler, eta, top)
        s0 = timesteps - 1
        prev_defer = dyn.defer_status_check
        dyn.defer_status_check = True
        try:
            g = self._graph(st, sampler, z_lig, xh_pocket, s0)
            self._start(st, z_lig, xh_pocket, s0)
            for s in reversed(range(timesteps)):
                g.replay()
                if (s * return_frames) % timesteps == 0:
                    idx = (s * return_frames) // timesteps
                    out_lig[idx], out_pocket[idx] = self.unnormalize_z(st['z'], st['pocket'])
        finally:
            dyn.defer_status_check = prev_defer
        dyn.check_status()
        return st['z'].clone(), st['pocket'].clone()

    def _fast_step(self, s, t, row, z_lig, xh_pocket, hist, lig_mask, pocket_mask, sampler, eta, u=0, commit=True):
        """Eager step z_t -> z_s of any sampler (DESIGN §13, §15): 'ddpm' is sample_p_zs_given_zt at s = ``row`` (the s/T
        array) and t; for 'ddim' / 'dpmpp_2m' / 'dpmpp_3m' ``row`` [1, k] is the step's row of _fast_tables.  ``hist``: the
        history (_empty_history).  Returns (z_lig, xh_pocket, hist): with ``commit`` the history multistep_update writes, else
        the one given; either way moved by the step's ligand-COM removal, so that it stays in the pocket's frame.  ``u``: the
        resampling round of the seeded reverse draw (RePaint)."""
        if sampler == 'ddpm':
            self._draw_at(seeded.STAGE_LOOP, s, u, seeded.PURPOSE_REVERSE)
            return (*self.sample_p_zs_given_zt(row, t, z_lig, xh_pocket, lig_mask, pocket_mask), hist)
        nd = self.n_dims
        c = row.expand(t.shape[0], -1)
        cl = c[lig_mask]
        eps, _ = self.dynamics(z_lig, xh_pocket, t, lig_mask, pocket_mask)
        if sampler == 'ddim':
            mu = z_lig / cl[:, 0:1] - cl[:, 1:2] * eps
            if eta > 0:
                self._draw_at(seeded.STAGE_LOOP, s, u, seeded.PURPOSE_REVERSE)
                z_lig, xh_pocket = self.sample_normal_zero_com(mu, xh_pocket, c[:, 2:3], lig_mask, pocket_mask)
            else:
                xh_pocket = xh_pocket.clone()
                mu[:, :nd], xh_pocket[:, :nd] = self.remove_mean_batch(mu[:, :nd], xh_pocket[:, :nd], lig_mask, pocket_mask)
                z_lig = mu
            return z_lig, xh_pocket, hist
        z_lig, new = multistep_update(z_lig, eps, hist, cl)
        hist = new if commit else tuple(h.clone() for h in hist)
        # the ligand COM leaves z, the pocket and the history together (one mean, subtracted from all)
        NP, NL = xh_pocket.shape[0], z_lig.shape[0]
        xh_pocket = xh_pocket.clone()
        z_lig[:, :nd], moved = self.remove_mean_batch(
            z_lig[:, :nd], torch.cat((xh_pocket[:, :nd],) + tuple(h[:, :nd] for h in hist)), lig_mask,
            torch.cat((pocket_mask,) + (lig_mask,) * len(hist)))
        xh_pocket[:, :nd] = moved[:NP]
        for k, h in enumerate(hist):
            h[:, :nd] = moved[NP + k * NL:NP + (k + 1) * NL]
        return z_lig, xh_pocket, hist

    def _fast_inpaint_step(self, s, u, t, row, gamma_s, gamma_t, z_lig, xh_pocket, hist, ligand_x, xh_ligand, com_pocket_0,
                           lig_fixed, lmask, pmask, sampler, eta, last):
        """Eager RePaint round (s, u) of _inpaint (DESIGN §14): the reverse step (_fast_step with ``t`` and ``row``), then
        the known part, the COM alignment, the blend and, unless ``last``, the re-noising.  ``hist`` (_empty_history) is the
        history committed by the last round of step s + 1, kept in the pocket's frame: every translation of the pocket
        coordinates moves it too, and the last round of step s commits its own (multistep_update); 'ddpm' and DDIM leave it
        as it is.  Returns (z_lig, xh_pocket, hist)."""
        nd, NL, NP = self.n_dims, z_lig.shape[0], xh_pocket.shape[0]
        fixed_rows = lig_fixed.bool().view(-1)
        z_unknown, xh_pocket, hist = self._fast_step(s, t, row, z_lig, xh_pocket, hist, lmask, pmask, sampler, eta, u, last)
        # frame: the rows that every pocket translation moves (the pocket's x columns and the history), under the pocket's
        # graph index
        frame = torch.cat((xh_pocket[:, :nd],) + tuple(h[:, :nd] for h in hist))
        fmask = torch.cat((pmask,) + (lmask,) * len(hist))

        # noise the known part to level s, following the pocket's current COM (conditional_model.py:636-643)
        com_pocket = scatter_mean(frame[:NP], pmask, dim=0)
        xh_ligand[:, :nd] = ligand_x + (com_pocket - com_pocket_0)[lmask]
        self._draw_at(seeded.STAGE_LOOP, s, u, seeded.PURPOSE_KNOWN)
        z_known, frame, _ = self.noised_representation(xh_ligand, frame, lmask, fmask, gamma_s)
        # align COM of the fixed atoms: noised -> denoised (conditional_model.py:645-656)
        com_noised = scatter_mean(z_known[fixed_rows][:, :nd], lmask[fixed_rows], dim=0)
        com_denoised = scatter_mean(z_unknown[fixed_rows][:, :nd], lmask[fixed_rows], dim=0)
        dx = com_denoised - com_noised
        z_known[:, :nd] = z_known[:, :nd] + dx[lmask]
        frame = frame + dx[fmask]
        z_lig = z_known * lig_fixed + z_unknown * (1 - lig_fixed)
        if not last:
            self._draw_at(seeded.STAGE_LOOP, s, u, seeded.PURPOSE_RENOISE)
            z_lig, frame = self.sample_p_zt_given_zs(z_lig, frame, lmask, fmask, gamma_t, gamma_s)
        xh_pocket = torch.cat((frame[:NP], xh_pocket[:, nd:]), dim=1)
        hist = tuple(torch.cat((frame[NP + k * NL:NP + (k + 1) * NL], h[:, nd:]), dim=1) for k, h in enumerate(hist))
        return z_lig, xh_pocket, hist

    def _graphed_inpaint_loop(self, z_lig, xh_pocket, xh_known, com_pocket_0, lig_fixed, lmask, pmask, n_samples,
                              timesteps, resamplings, return_frames, out_lig, out_pocket, sampler='ddpm', eta=0.0):
        """The double loop of conditional_model.py:616-674 as graph replays: per (s, u) one captured graph = native
        denoiser + fused reverse update + fused RePaint iteration (dsb_ddpm_inpaint_update, or one
        dsb_ddpm_multistep_inpaint_update under 2M); no torch op and no host sync inside the loop."""
        dyn: EGNNDynamics = self.dynamics
        st = self._engine(z_lig, xh_pocket, lmask, pmask, n_samples, timesteps, self._seeds(), sampler, eta)
        if st['inpaint'] is None:       # static buffers the captured RePaint iteration reads
            st['inpaint'] = dict(known=torch.empty_like(z_lig), com0=torch.empty_like(com_pocket_0, dtype=torch.float32),
                                 fixed=torch.empty(z_lig.shape[0], dtype=torch.float32, device=z_lig.device))
        ip = st['inpaint']
        ip['known'].copy_(xh_known); ip['com0'].copy_(com_pocket_0); ip['fixed'].copy_(lig_fixed.reshape(-1))
        prev_defer = dyn.defer_status_check
        dyn.defer_status_check = True
        s0 = timesteps - 1
        try:
            g_last = self._graph(st, 'inpaint_last', z_lig, xh_pocket, s0)
            g_re = self._graph(st, 'inpaint_renoise', z_lig, xh_pocket, s0) if resamplings > 1 else None
            self._start(st, z_lig, xh_pocket, s0)
            for s in reversed(range(0, timesteps)):
                for _ in range(resamplings - 1):
                    g_re.replay()
                g_last.replay()
                if (s * return_frames) % timesteps == 0:
                    idx = (s * return_frames) // timesteps
                    out_lig[idx], out_pocket[idx] = self.unnormalize_z(st['z'], st['pocket'])
        finally:
            dyn.defer_status_check = prev_defer
        dyn.check_status()
        return st['z'].clone(), st['pocket'].clone()

    # ---- public samplers ------------------------------------------------------------------------------------
    @follows_dynamics_determinism
    @torch.no_grad()
    def sample_given_pocket(self, pocket, num_nodes_lig, return_frames=1, timesteps=None, seeds=None, sampler='ddpm', eta=0.0):
        """conditional_model.py:479-555.  ``seeds``: one int64 per sample (seeded.py); every draw then comes from the
        sample's own seed instead of torch's global generator.  ``sampler``: 'ddpm' (the reference's ancestral step),
        'ddim' (with noise level ``eta`` in [0, 1]), 'dpmpp_2m' or 'dpmpp_3m', on the same ``timesteps`` grid (DESIGN §13,
        §15)."""
        check_sampler(sampler, eta)
        timesteps = self.T if timesteps is None else timesteps
        assert 0 < return_frames <= timesteps
        assert timesteps % return_frames == 0
        n_samples = len(pocket['size'])
        device = pocket['x'].device
        seeds = seeded.as_seeds(seeds, n_samples, device)
        lig_mask = num_nodes_to_batch_mask(n_samples, num_nodes_lig, device)
        with self._seeded(seeds, lig_mask, pocket['mask']):
            return self._sample_given_pocket(pocket, lig_mask, n_samples, return_frames, timesteps, sampler, float(eta))

    def _sample_given_pocket(self, pocket, lig_mask, n_samples, return_frames, timesteps, sampler='ddpm', eta=0.0):
        if self._rng is not None:
            seeded.check_schedule(timesteps)
        device = pocket['x'].device
        _, pocket = self.normalize(pocket=pocket)
        xh0_pocket = torch.cat([pocket['x'], pocket['one_hot']], dim=1)

        # ligand prior centred on the pocket COM (conditional_model.py:501-510)
        mu_lig_x = scatter_mean(pocket['x'], pocket['mask'], dim=0)
        mu_lig_h = torch.zeros((n_samples, self.atom_nf), device=device)
        mu_lig = torch.cat((mu_lig_x, mu_lig_h), dim=1)[lig_mask]
        sigma = torch.ones_like(pocket['size']).unsqueeze(1)
        self._draw_at(seeded.STAGE_PRIOR)
        z_lig, xh_pocket = self.sample_normal_zero_com(mu_lig, xh0_pocket, sigma, lig_mask, pocket['mask'])
        self.assert_mean_zero_with_mask(z_lig[:, :self.n_dims], lig_mask)

        out_lig = torch.zeros((return_frames,) + z_lig.size(), device=z_lig.device)
        out_pocket = torch.zeros((return_frames,) + xh_pocket.size(), device=device)

        use_graph = self._use_graph(device)
        if use_graph and sampler != 'ddpm':
            z_lig, xh_pocket = self._graphed_fast_loop(z_lig, xh_pocket, lig_mask, pocket['mask'], n_samples, timesteps, sampler,
                                                       eta, return_frames, out_lig, out_pocket)
        elif use_graph:
            stride = timesteps // return_frames       # frames are saved at s = idx * stride
            s_hi = timesteps - 1
            while s_hi >= 0:
                s_lo = (s_hi // stride) * stride
                z_lig, xh_pocket = self._graphed_reverse_steps(
                    z_lig, xh_pocket, lig_mask, pocket['mask'], n_samples, s_hi, s_hi - s_lo + 1, timesteps)
                out_lig[s_lo // stride], out_pocket[s_lo // stride] = self.unnormalize_z(z_lig, xh_pocket)
                s_hi = s_lo - 1
        else:
            fast = None if sampler == 'ddpm' else self._fast_tables(timesteps, sampler, eta, device)
            hist = self._empty_history(z_lig, sampler)
            for s in reversed(range(0, timesteps)):
                t, row = self._eager_row(s, timesteps, n_samples, device, fast)
                z_lig, xh_pocket, hist = self._fast_step(s, t, row, z_lig, xh_pocket, hist, lig_mask, pocket['mask'], sampler,
                                                         eta)
                if (s * return_frames) % timesteps == 0:
                    idx = (s * return_frames) // timesteps
                    out_lig[idx], out_pocket[idx] = self.unnormalize_z(z_lig, xh_pocket)
        self.assert_mean_zero_with_mask(z_lig[:, :self.n_dims], lig_mask)

        self._draw_at(seeded.STAGE_FINAL)
        x_lig, h_lig, x_pocket, h_pocket = self.sample_p_xh_given_z0(z_lig, xh_pocket, lig_mask, pocket['mask'], n_samples)
        self.assert_mean_zero_with_mask(x_lig, lig_mask)
        if return_frames == 1:                          # conditional_model.py:540-547
            x_lig, x_pocket = self._project_cog_drift(
                x_lig, x_pocket, lig_mask, lambda: self.remove_mean_batch(x_lig, x_pocket, lig_mask, pocket['mask']),
                pocket['mask'])
        out_lig[0] = torch.cat([x_lig, h_lig], dim=1)
        out_pocket[0] = torch.cat([x_pocket, h_pocket], dim=1)
        return out_lig.squeeze(0), out_pocket.squeeze(0), lig_mask, pocket['mask']

    @follows_dynamics_determinism
    @torch.no_grad()
    def inpaint(self, ligand, pocket, lig_fixed, resamplings=1, return_frames=1, timesteps=None, center='ligand', seeds=None,
                sampler='ddpm', eta=0.0):
        """conditional_model.py:558-686: RePaint-style conditional generation with fixed ligand atoms.  ``seeds``: as
        sample_given_pocket.  ``sampler`` / ``eta``: the reverse step of every RePaint round, as sample_given_pocket
        (DESIGN §14)."""
        self._check_fast_repaint(sampler, eta)
        seeds = seeded.as_seeds(seeds, len(ligand['size']), pocket['x'].device)
        with self._seeded(seeds, ligand['mask'], pocket['mask']):
            return self._inpaint(ligand, pocket, lig_fixed, resamplings, return_frames, timesteps, center, sampler, float(eta))

    def _check_fast_repaint(self, sampler, eta):
        check_sampler(sampler, eta)

    def _inpaint(self, ligand, pocket, lig_fixed, resamplings, return_frames, timesteps, center, sampler='ddpm', eta=0.0):
        timesteps = self.T if timesteps is None else timesteps
        if self._rng is not None:
            seeded.check_schedule(timesteps, resamplings)
        assert 0 < return_frames <= timesteps
        assert timesteps % return_frames == 0
        if len(lig_fixed.size()) == 1:
            lig_fixed = lig_fixed.unsqueeze(1)
        n_samples = len(ligand['size'])
        device = pocket['x'].device
        ligand, pocket = self.normalize(ligand, pocket)
        lmask, pmask = ligand['mask'], pocket['mask']
        fixed_rows = lig_fixed.bool().view(-1)

        xh0_pocket = torch.cat([pocket['x'], pocket['one_hot']], dim=1)
        com_pocket_0 = scatter_mean(pocket['x'], pmask, dim=0)
        xh_ligand = torch.cat([ligand['x'], ligand['one_hot']], dim=1).clone()
        if center == 'ligand':
            mean_known = scatter_mean(ligand['x'][fixed_rows], lmask[fixed_rows], dim=0)
        elif center == 'pocket':
            mean_known = scatter_mean(pocket['x'], pmask, dim=0)
        else:
            raise NotImplementedError(f"Centering option {center} not implemented")

        mu_lig = torch.cat((mean_known, torch.zeros((n_samples, self.atom_nf), device=device)), dim=1)[lmask]
        sigma = torch.ones_like(pocket['size']).unsqueeze(1)
        self._draw_at(seeded.STAGE_PRIOR)
        z_lig, xh_pocket = self.sample_normal_zero_com(mu_lig, xh0_pocket, sigma, lmask, pmask)

        out_lig = torch.zeros((return_frames,) + z_lig.size(), device=z_lig.device)
        out_pocket = torch.zeros((return_frames,) + xh_pocket.size(), device=device)
        if self._use_graph(device):
            z_lig, xh_pocket = self._graphed_inpaint_loop(z_lig, xh_pocket, xh_ligand, com_pocket_0, lig_fixed, lmask, pmask,
                                                         n_samples, timesteps, resamplings, return_frames, out_lig, out_pocket,
                                                         sampler, eta)
        else:
            if sampler != 'ddpm':
                t_table, coef = self._fast_tables(timesteps, sampler, eta, device)
            hist = self._empty_history(z_lig, sampler)
            for s in reversed(range(0, timesteps)):
                for u in range(resamplings):
                    s_array = torch.full((n_samples, 1), fill_value=s, device=device)
                    t_array = (s_array + 1) / timesteps
                    s_array = s_array / timesteps
                    last = u == resamplings - 1
                    t, row = (t_array, s_array) if sampler == 'ddpm' else (t_table[s].expand(n_samples, 1), coef[s:s + 1])
                    z_lig, xh_pocket, hist = self._fast_inpaint_step(
                        s, u, t, row, self.gamma(s_array), self.gamma(t_array), z_lig, xh_pocket, hist, ligand['x'], xh_ligand,
                        com_pocket_0, lig_fixed, lmask, pmask, sampler, eta, last)
                    if last and (s * return_frames) % timesteps == 0:
                        idx = (s * return_frames) // timesteps
                        out_lig[idx], out_pocket[idx] = self.unnormalize_z(z_lig, xh_pocket)

        self._draw_at(seeded.STAGE_FINAL)
        x_lig, h_lig, x_pocket, h_pocket = self.sample_p_xh_given_z0(z_lig, xh_pocket, lmask, pmask, n_samples)
        out_lig[0] = torch.cat([x_lig, h_lig], dim=1)
        out_pocket[0] = torch.cat([x_pocket, h_pocket], dim=1)
        return out_lig.squeeze(0), out_pocket.squeeze(0), lmask, pmask

    # ---- evaluation-mode variational bound (conditional_model.py:20-110, :185-330) ---------------------------------------
    def log_pN(self, N_lig, N_pocket):
        """log p(N_lig | N_pocket): the ligand size prior given the pocket."""
        return self.size_distribution.log_prob_n1_given_n2(N_lig, N_pocket)

    def kl_prior(self, xh_lig, mask_lig, num_nodes):
        """conditional_model.py:20-56: KL of q(z_T | x, h) of the ligand against the standard normal prior."""
        nd = self.n_dims
        alpha_T = self.alpha(self.gamma(torch.ones((len(num_nodes), 1), device=xh_lig.device)), xh_lig)
        mu = alpha_T[mask_lig] * xh_lig
        return self._kl_prior_from_norms(self.sum_except_batch(mu[:, :nd] ** 2, mask_lig),
                                         self.sum_except_batch(mu[:, nd:] ** 2, mask_lig), num_nodes, xh_lig.device)

    def _virtual_rows(self, ligand):
        return ligand['one_hot'][:, self.vnode_idx].bool()

    def log_pxh_given_z0_without_constants(self, ligand, z_0_lig, eps_lig, net_out_lig, gamma_0, epsilon=1e-10):
        """conditional_model.py:58-110: -1/2 |eps_0.x - net_0.x|^2 (virtual atoms excluded) and log p(h | z_0), ligand only."""
        nd = self.n_dims
        sigma_0_cat = self.sigma(gamma_0, target_tensor=z_0_lig) * self.norm_values[1]
        sq = (eps_lig[:, :nd] - net_out_lig[:, :nd]) ** 2
        if self.vnode_idx is not None:
            sq[self._virtual_rows(ligand)] = 0
        log_px = -0.5 * self.sum_except_batch(sq, ligand['mask'])
        return log_px, self._log_ph_given_z0(ligand['one_hot'], z_0_lig[:, nd:], sigma_0_cat, ligand['mask'], epsilon)

    def _native_noise_conditional(self, xh_lig, eps, xh_pocket, lig_mask, pocket_mask, gamma):
        """q(z_t | x, h) with the ligand COM removed from z and pocket (:162-183) as one dsb_ddpm_ligand_update launch:
        coef = (1/alpha, 0, sigma) turns its z/alpha_ts - coef1 eps_hat + sigma noise into alpha xh + sigma eps."""
        lib = _native.load()
        alpha, sigma = self.alpha(gamma, gamma), self.sigma(gamma, gamma)
        coef = torch.cat([1. / alpha, torch.zeros_like(alpha), sigma], dim=1).float().contiguous()
        z, pocket_out = torch.empty_like(xh_lig), torch.empty_like(xh_pocket)
        _native.check(lib.dsb_ddpm_ligand_update(
            xh_lig.data_ptr(), eps.data_ptr(), eps.data_ptr(), coef.data_ptr(), lig_mask.data_ptr(), pocket_mask.data_ptr(),
            xh_pocket.data_ptr(), len(lig_mask), len(pocket_mask), coef.shape[0], self.atom_nf, self.residue_nf,
            z.data_ptr(), pocket_out.data_ptr(), C.c_void_p(torch.cuda.current_stream(xh_lig.device).cuda_stream)))
        return z, pocket_out

    @follows_dynamics_determinism
    @torch.no_grad()
    def forward(self, ligand, pocket, return_info=False):
        """Eval-mode variational bound (conditional_model.py:202-330): the terms of -log p(x, h | N, pocket) of the ligand
        at one random t in [1, T] plus the t = 0 reconstruction term, with the reference's RNG call order (randint for t,
        noise at t, noise at 0).  Training (t = 0 sampling, autograd) is not built."""
        if self.training:
            raise NotImplementedError('the training loss is not built (no backward kernels); call eval() for the NLL bound')
        ligand, pocket = self.normalize(ligand, pocket)
        lm, pm = ligand['mask'], pocket['mask']
        n, device, nd = ligand['size'].size(0), ligand['x'].device, self.n_dims
        delta_log_px = self.delta_log_px(ligand['size'])
        t_int = torch.randint(1, self.T + 1, size=(n, 1), device=device).float()
        s, t = (t_int - 1) / self.T, t_int / self.T
        t_0 = torch.zeros_like(s)
        gamma_s = self.inflate_batch_array(self.gamma(s), ligand['x'])
        gamma_t = self.inflate_batch_array(self.gamma(t), ligand['x'])
        gamma_0 = self.inflate_batch_array(self.gamma(t_0), ligand['x'])
        xh0_lig = torch.cat([ligand['x'], ligand['one_hot']], dim=1)
        xh0_pocket = torch.cat([pocket['x'], pocket['one_hot']], dim=1)
        xh0_lig[:, :nd], xh0_pocket[:, :nd] = self.remove_mean_batch(xh0_lig[:, :nd], xh0_pocket[:, :nd], lm, pm)
        SNR_weight = (1 - self.SNR(gamma_s - gamma_t)).squeeze(1)
        neg_log_constants = -self.log_constants_p_x_given_z0(n_nodes=ligand['size'], device=device)

        if self._vlb_native(device):
            size = (len(lm), nd + self.atom_nf)
            eps_t_lig = self.sample_gaussian(size=size, device=device)
            z_t = self._native_noise_conditional(xh0_lig, eps_t_lig, xh0_pocket, lm, pm, gamma_t)
            eps_0_lig = self.sample_gaussian(size=size, device=device)
            z_0 = self._native_noise_conditional(xh0_lig, eps_0_lig, xh0_pocket, lm, pm, gamma_0)
            (net_t_lig, _), (net_0_lig, _) = self._native_denoise_pair(z_t, t, z_0, t_0, lm, pm)
            terms, xh_lig_hat = self._native_vlb_terms(
                (xh0_lig, z_t[0], eps_t_lig, net_t_lig, z_0[0], eps_0_lig, net_0_lig), None, lm, pm, gamma_t, gamma_0,
                self.vnode_idx)
            error_t_lig = terms[:, 0]
            loss_0_x_ligand, loss_0_h = 0.5 * terms[:, 2], -terms[:, 4]
            kl_prior = self._kl_prior_from_norms(terms[:, 5], terms[:, 6], ligand['size'], device)
            cnt = ligand['size'].clamp(min=1).float()
            info = {'eps_hat_lig_x': (terms[:, 7] / (nd * cnt)).mean(),
                    'eps_hat_lig_h': (terms[:, 8] / (self.atom_nf * cnt)).mean()}
        else:
            z_t_lig, xh_pocket_t, eps_t_lig = self.noised_representation(xh0_lig, xh0_pocket, lm, pm, gamma_t)
            net_t_lig, _ = self.dynamics(z_t_lig, xh_pocket_t, t, lm, pm)
            xh_lig_hat = self.xh_given_zt_and_epsilon(z_t_lig, net_t_lig, gamma_t, lm)
            sq = (eps_t_lig - net_t_lig) ** 2
            if self.vnode_idx is not None:
                sq[self._virtual_rows(ligand), :nd] = 0
            error_t_lig = self.sum_except_batch(sq, lm)
            kl_prior = self.kl_prior(xh0_lig, lm, ligand['size'])
            z_0_lig, xh_pocket_0, eps_0_lig = self.noised_representation(xh0_lig, xh0_pocket, lm, pm, gamma_0)
            net_0_lig, _ = self.dynamics(z_0_lig, xh_pocket_0, t_0, lm, pm)
            log_px, log_ph = self.log_pxh_given_z0_without_constants(ligand, z_0_lig, eps_0_lig, net_0_lig, gamma_0)
            loss_0_x_ligand, loss_0_h = -log_px, -log_ph
            info = {'eps_hat_lig_x': self._eps_hat_mean(net_t_lig[:, :nd], lm, n),
                    'eps_hat_lig_h': self._eps_hat_mean(net_t_lig[:, nd:], lm, n)}

        log_pN = self.log_pN(ligand['size'], pocket['size'])
        terms = (delta_log_px, error_t_lig, torch.tensor(0.0), SNR_weight, loss_0_x_ligand, torch.tensor(0.0), loss_0_h,
                 neg_log_constants, kl_prior, log_pN, t_int.squeeze(), xh_lig_hat)
        return (*terms, info) if return_info else terms

    def partially_noised_ligand(self, ligand, pocket, noising_steps):
        """conditional_model.py:332-362."""
        t = torch.ones(size=(ligand['size'].size(0), 1), device=ligand['x'].device).float() * noising_steps / self.T
        gamma_t = self.inflate_batch_array(self.gamma(t), ligand['x'])
        xh0_lig = torch.cat([ligand['x'], ligand['one_hot']], dim=1)
        xh0_pocket = torch.cat([pocket['x'], pocket['one_hot']], dim=1)
        xh0_lig[:, :self.n_dims], xh0_pocket[:, :self.n_dims] = self.remove_mean_batch(
            xh0_lig[:, :self.n_dims], xh0_pocket[:, :self.n_dims], ligand['mask'], pocket['mask'])
        return self.noised_representation(xh0_lig, xh0_pocket, ligand['mask'], pocket['mask'], gamma_t)

    @follows_dynamics_determinism
    @torch.no_grad()
    def diversify(self, ligand, pocket, noising_steps, seeds=None, sampler='ddpm', eta=0.0, denoising_steps=None):
        """conditional_model.py:364-409: partially noise given ligands, then denoise them again.  ``seeds``: as
        sample_given_pocket.  ``sampler`` / ``eta``: the reverse step, as sample_given_pocket; ``denoising_steps``: the
        number of reverse steps from t* = noising_steps / T down to 0 on the uniform grid t_k = k t* / denoising_steps,
        1 <= denoising_steps <= noising_steps (None: noising_steps, the T grid; 'ddpm' runs the T grid only) (DESIGN §14)."""
        self._check_fast_repaint(sampler, eta)
        if denoising_steps is not None:
            if int(denoising_steps) != denoising_steps or not 1 <= denoising_steps <= noising_steps:
                raise ValueError(f'denoising_steps must be an integer in [1, noising_steps = {noising_steps}], '
                                 f'got {denoising_steps}')
            if sampler == 'ddpm' and denoising_steps != noising_steps:
                raise ValueError(f"sampler='ddpm' denoises on the T grid: denoising_steps must be None or noising_steps "
                                 f"({noising_steps}), got {denoising_steps}; use sampler='ddim' or 'dpmpp_2m' for fewer steps")
        seeds = seeded.as_seeds(seeds, len(pocket['size']), pocket['x'].device)
        with self._seeded(seeds, ligand['mask'], pocket['mask']):
            return self._diversify(ligand, pocket, noising_steps, sampler, float(eta),
                                   noising_steps if denoising_steps is None else int(denoising_steps))

    def _diversify(self, ligand, pocket, noising_steps, sampler='ddpm', eta=0.0, denoising_steps=None):
        if self._rng is not None:
            seeded.check_schedule(self.T)
        ligand, pocket = self.normalize(ligand, pocket)
        self._draw_at(seeded.STAGE_PARTIAL)
        z_lig, xh_pocket, _ = self.partially_noised_ligand(ligand, pocket, noising_steps)
        timesteps = self.T
        n_samples = len(pocket['size'])
        lig_mask = ligand['mask']
        self.assert_mean_zero_with_mask(z_lig[:, :self.n_dims], lig_mask)
        top = (noising_steps, timesteps)
        device = z_lig.device
        use_graph = self._use_graph(device) and noising_steps > 0
        if use_graph and sampler != 'ddpm':
            frame = torch.empty((1,) + z_lig.shape, device=device), torch.empty((1,) + xh_pocket.shape, device=device)
            z_lig, xh_pocket = self._graphed_fast_loop(z_lig, xh_pocket, lig_mask, pocket['mask'], n_samples, denoising_steps,
                                                       sampler, eta, 1, *frame, top=top)
        elif use_graph:
            z_lig, xh_pocket = self._graphed_reverse_steps(z_lig, xh_pocket, lig_mask, pocket['mask'], n_samples,
                                                           noising_steps - 1, noising_steps, timesteps)
        elif noising_steps > 0:           # 'ddpm' takes the T grid: denoising_steps = noising_steps
            fast = None if sampler == 'ddpm' else self._fast_tables(denoising_steps, sampler, eta, device, top)
            hist = self._empty_history(z_lig, sampler)
            for s in reversed(range(0, denoising_steps)):
                t, row = self._eager_row(s, timesteps, n_samples, device, fast)
                z_lig, xh_pocket, hist = self._fast_step(s, t, row, z_lig, xh_pocket, hist, lig_mask, pocket['mask'], sampler,
                                                         eta)
        self._draw_at(seeded.STAGE_FINAL)
        x_lig, h_lig, x_pocket, h_pocket = self.sample_p_xh_given_z0(z_lig, xh_pocket, lig_mask, pocket['mask'], n_samples)
        self.assert_mean_zero_with_mask(x_lig, lig_mask)
        return torch.cat([x_lig, h_lig], dim=1), torch.cat([x_pocket, h_pocket], dim=1), lig_mask, pocket['mask']


class SimpleConditionalDDPM(ConditionalDDPM):
    """conditional_model.py:702-746: the conditional model without the COM-free subspace trick."""

    def subspace_dimensionality(self, input_size):
        return input_size * self.n_dims

    @classmethod
    def remove_mean_batch(cls, x_lig, x_pocket, lig_indices, pocket_indices):
        return x_lig, x_pocket

    @staticmethod
    def assert_mean_zero_with_mask(x, node_mask, eps=1e-10):
        return

    def _use_graph(self, device) -> bool:
        return False    # the fused update kernel hard-wires the COM projection of ConditionalDDPM

    def _native_noise_conditional(self, xh_lig, eps, xh_pocket, lig_mask, pocket_mask, gamma):
        z_lig, _ = self._native_noise(xh_lig, eps, None, None, lig_mask, pocket_mask, gamma)   # no COM projection
        return z_lig, xh_pocket

    def _check_fast_repaint(self, sampler, eta):
        check_sampler(sampler, eta)
        if sampler != 'ddpm':
            raise ValueError(f"sampler={sampler!r}: inpaint and diversify of SimpleConditionalDDPM run the 'ddpm' step only")

    @follows_dynamics_determinism
    def forward(self, ligand, pocket, return_info=False):
        """conditional_model.py:727-735: the likelihood is evaluated in the frame of the pocket's centre of mass."""
        pocket_com = scatter_mean(pocket['x'], pocket['mask'], dim=0)
        ligand['x'] = ligand['x'] - pocket_com[ligand['mask']]
        pocket['x'] = pocket['x'] - pocket_com[pocket['mask']]
        return super().forward(ligand, pocket, return_info)

    @follows_dynamics_determinism
    @torch.no_grad()
    def sample_given_pocket(self, pocket, num_nodes_lig, return_frames=1, timesteps=None, seeds=None, sampler='ddpm', eta=0.0):
        check_sampler(sampler, eta)
        pocket_com = scatter_mean(pocket['x'], pocket['mask'], dim=0)
        pocket['x'] = pocket['x'] - pocket_com[pocket['mask']]
        return super().sample_given_pocket(pocket, num_nodes_lig, return_frames, timesteps, seeds, sampler, eta)
