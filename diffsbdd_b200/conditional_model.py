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

from . import _native
from .dynamics import EGNNDynamics
from .en_diffusion import EnVariationalDiffusion, follows_dynamics_determinism, scatter_add, scatter_mean, num_nodes_to_batch_mask


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
        eps = self.sample_gaussian(size=(len(lig_mask), self.n_dims + self.atom_nf), device=lig_mask.device)
        out_lig = mu_lig + sigma[lig_mask] * eps
        xh_pocket = xh0_pocket.detach().clone()
        out_lig[:, :self.n_dims], xh_pocket[:, :self.n_dims] = self.remove_mean_batch(
            out_lig[:, :self.n_dims], xh0_pocket[:, :self.n_dims], lig_mask, pocket_mask)
        return out_lig, xh_pocket

    def noised_representation(self, xh_lig, xh0_pocket, lig_mask, pocket_mask, gamma_t):
        """conditional_model.py:162-183: z_t ~ q(z_t | x, h) for the ligand; pocket follows the COM shift."""
        alpha_t, sigma_t = self.alpha(gamma_t, xh_lig), self.sigma(gamma_t, xh_lig)
        eps = self.sample_gaussian(size=(len(lig_mask), self.n_dims + self.atom_nf), device=lig_mask.device)
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

    def _engine(self, z_lig, xh_pocket, lig_mask, pocket_mask, n_samples, timesteps):
        """Static buffers + captured graphs for one batch layout.  A cached engine is reused only while everything a
        captured graph bakes in is unchanged: batch layout (mask contents), the native module generation (packed-weight
        blob), its arithmetic mode and its workspace/status buffers."""
        device = z_lig.device
        dyn: EGNNDynamics = self.dynamics
        dyn._ensure_handle(device)
        key = (tuple(z_lig.shape), tuple(xh_pocket.shape), n_samples, timesteps, str(device))
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
                n_samples=n_samples, inpaint=None)
            self._graph_cache[key] = st
        return st

    def _captured_step(self, st, kind):
        """One iteration as a python callable over the static buffers of ``st``.
        kind: 'reverse' (z_t -> z_s, step -= 1) | 'inpaint_renoise' (reverse step + RePaint blend + re-noise to t) |
        'inpaint_last' (reverse step + blend, step -= 1)."""
        dyn: EGNNDynamics = self.dynamics
        lib = _native.load()
        lm, pm, n = st['lig_mask'], st['pocket_mask'], st['n_samples']
        NL, NP = st['z'].shape[0], st['pocket'].shape[0]

        def run():
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            idx = st['step'].clamp(min=0)
            st['t'].copy_(st['t_table'].index_select(0, idx).expand(n, 1))
            row = st['coef_table'].index_select(0, idx)
            st['coef3'].copy_(row[:, :3].expand(n, 3))
            st['coef4'].copy_(row[:, 3:].expand(n, 4))
            eps, _ = dyn(st['z'], st['pocket'], st['t'], lm, pm)
            st['noise'].normal_()
            _native.check(lib.dsb_ddpm_ligand_update(
                st['z'].data_ptr(), eps.data_ptr(), st['noise'].data_ptr(), st['coef3'].data_ptr(),
                lm.data_ptr(), pm.data_ptr(), st['pocket'].data_ptr(), NL, NP, n, self.atom_nf, self.residue_nf,
                st['z'].data_ptr(), st['pocket'].data_ptr(), stream))
            if kind != 'reverse':
                ip = st['inpaint']
                st['noise1'].normal_()
                renoise = kind == 'inpaint_renoise'
                if renoise:
                    st['noise2'].normal_()
                _native.check(lib.dsb_ddpm_inpaint_update(
                    st['z'].data_ptr(), st['pocket'].data_ptr(), ip['known'].data_ptr(), ip['com0'].data_ptr(),
                    ip['fixed'].data_ptr(), st['noise1'].data_ptr(), st['noise2'].data_ptr() if renoise else None,
                    st['coef4'].data_ptr(), lm.data_ptr(), pm.data_ptr(), NL, NP, n, self.atom_nf, self.residue_nf, stream))
            if kind != 'inpaint_renoise':
                st['step'].sub_(1)
        return run

    def _graph(self, st, kind, z_lig, xh_pocket, first_s):
        """Captured CUDA graph of ``kind`` (captured on first use; capture leaves the static state as it found it)."""
        g = st['graphs'].get(kind)
        if g is not None:
            return g
        device = z_lig.device
        dyn: EGNNDynamics = self.dynamics
        run = self._captured_step(st, kind)

        def reset():
            st['z'].copy_(z_lig); st['pocket'].copy_(xh_pocket); st['step'].fill_(first_s)

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
        st = self._engine(z_lig, xh_pocket, lig_mask, pocket_mask, n_samples, timesteps)
        prev_defer = dyn.defer_status_check
        dyn.defer_status_check = True
        try:
            g = self._graph(st, 'reverse', z_lig, xh_pocket, first_s)
            st['z'].copy_(z_lig); st['pocket'].copy_(xh_pocket); st['step'].fill_(first_s)
            for _ in range(n_steps):
                g.replay()
        finally:
            dyn.defer_status_check = prev_defer
        dyn.check_status()
        return st['z'].clone(), st['pocket'].clone()

    def _graphed_inpaint_loop(self, z_lig, xh_pocket, xh_known, com_pocket_0, lig_fixed, lmask, pmask, n_samples,
                              timesteps, resamplings, return_frames, out_lig, out_pocket):
        """The double loop of conditional_model.py:616-674 as graph replays: per (s, u) one captured graph = native
        denoiser + fused reverse update + fused RePaint iteration (dsb_ddpm_inpaint_update); no torch op and no host
        sync inside the loop."""
        dyn: EGNNDynamics = self.dynamics
        st = self._engine(z_lig, xh_pocket, lmask, pmask, n_samples, timesteps)
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
            st['z'].copy_(z_lig); st['pocket'].copy_(xh_pocket); st['step'].fill_(s0)
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
    def sample_given_pocket(self, pocket, num_nodes_lig, return_frames=1, timesteps=None):
        """conditional_model.py:479-555."""
        timesteps = self.T if timesteps is None else timesteps
        assert 0 < return_frames <= timesteps
        assert timesteps % return_frames == 0
        n_samples = len(pocket['size'])
        device = pocket['x'].device
        _, pocket = self.normalize(pocket=pocket)
        xh0_pocket = torch.cat([pocket['x'], pocket['one_hot']], dim=1)
        lig_mask = num_nodes_to_batch_mask(n_samples, num_nodes_lig, device)

        # ligand prior centred on the pocket COM (conditional_model.py:501-510)
        mu_lig_x = scatter_mean(pocket['x'], pocket['mask'], dim=0)
        mu_lig_h = torch.zeros((n_samples, self.atom_nf), device=device)
        mu_lig = torch.cat((mu_lig_x, mu_lig_h), dim=1)[lig_mask]
        sigma = torch.ones_like(pocket['size']).unsqueeze(1)
        z_lig, xh_pocket = self.sample_normal_zero_com(mu_lig, xh0_pocket, sigma, lig_mask, pocket['mask'])
        self.assert_mean_zero_with_mask(z_lig[:, :self.n_dims], lig_mask)

        out_lig = torch.zeros((return_frames,) + z_lig.size(), device=z_lig.device)
        out_pocket = torch.zeros((return_frames,) + xh_pocket.size(), device=device)

        if self._use_graph(device):
            stride = timesteps // return_frames       # frames are saved at s = idx * stride
            s_hi = timesteps - 1
            while s_hi >= 0:
                s_lo = (s_hi // stride) * stride
                z_lig, xh_pocket = self._graphed_reverse_steps(
                    z_lig, xh_pocket, lig_mask, pocket['mask'], n_samples, s_hi, s_hi - s_lo + 1, timesteps)
                out_lig[s_lo // stride], out_pocket[s_lo // stride] = self.unnormalize_z(z_lig, xh_pocket)
                s_hi = s_lo - 1
            self.assert_mean_zero_with_mask(z_lig[:, :self.n_dims], lig_mask)
        else:
            for s in reversed(range(0, timesteps)):
                s_array = torch.full((n_samples, 1), fill_value=s, device=z_lig.device)
                t_array = (s_array + 1) / timesteps
                s_array = s_array / timesteps
                z_lig, xh_pocket = self.sample_p_zs_given_zt(s_array, t_array, z_lig, xh_pocket, lig_mask, pocket['mask'])
                if (s * return_frames) % timesteps == 0:
                    idx = (s * return_frames) // timesteps
                    out_lig[idx], out_pocket[idx] = self.unnormalize_z(z_lig, xh_pocket)

        x_lig, h_lig, x_pocket, h_pocket = self.sample_p_xh_given_z0(z_lig, xh_pocket, lig_mask, pocket['mask'], n_samples)
        self.assert_mean_zero_with_mask(x_lig, lig_mask)
        if return_frames == 1:                          # conditional_model.py:540-547
            max_cog = scatter_add(x_lig, lig_mask, dim=0).abs().max().item()
            if max_cog > 5e-2:
                print(f'Warning CoG drift with error {max_cog:.3f}. Projecting the positions down.')
                x_lig, x_pocket = self.remove_mean_batch(x_lig, x_pocket, lig_mask, pocket['mask'])
        out_lig[0] = torch.cat([x_lig, h_lig], dim=1)
        out_pocket[0] = torch.cat([x_pocket, h_pocket], dim=1)
        return out_lig.squeeze(0), out_pocket.squeeze(0), lig_mask, pocket['mask']

    @follows_dynamics_determinism
    @torch.no_grad()
    def inpaint(self, ligand, pocket, lig_fixed, resamplings=1, return_frames=1, timesteps=None, center='ligand'):
        """conditional_model.py:558-686: RePaint-style conditional generation with fixed ligand atoms."""
        timesteps = self.T if timesteps is None else timesteps
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
        z_lig, xh_pocket = self.sample_normal_zero_com(mu_lig, xh0_pocket, sigma, lmask, pmask)

        out_lig = torch.zeros((return_frames,) + z_lig.size(), device=z_lig.device)
        out_pocket = torch.zeros((return_frames,) + xh_pocket.size(), device=device)
        use_graph = self._use_graph(device)
        nd = self.n_dims

        if use_graph:
            z_lig, xh_pocket = self._graphed_inpaint_loop(z_lig, xh_pocket, xh_ligand, com_pocket_0, lig_fixed, lmask, pmask,
                                                         n_samples, timesteps, resamplings, return_frames, out_lig, out_pocket)
        else:
            for s in reversed(range(0, timesteps)):
                for u in range(resamplings):
                    s_array = torch.full((n_samples, 1), fill_value=s, device=device)
                    t_array = (s_array + 1) / timesteps
                    s_array = s_array / timesteps
                    gamma_t, gamma_s = self.gamma(t_array), self.gamma(s_array)

                    # denoise the whole ligand one step (unknown part)
                    z_unknown, xh_pocket = self.sample_p_zs_given_zt(s_array, t_array, z_lig, xh_pocket, lmask, pmask)

                    # noise the known part to level s, following the pocket's current COM (conditional_model.py:636-643)
                    com_pocket = scatter_mean(xh_pocket[:, :nd], pmask, dim=0)
                    xh_ligand[:, :nd] = ligand['x'] + (com_pocket - com_pocket_0)[lmask]
                    z_known, xh_pocket, _ = self.noised_representation(xh_ligand, xh_pocket, lmask, pmask, gamma_s)

                    # align COM of the fixed atoms: noised -> denoised (conditional_model.py:645-656)
                    com_noised = scatter_mean(z_known[fixed_rows][:, :nd], lmask[fixed_rows], dim=0)
                    com_denoised = scatter_mean(z_unknown[fixed_rows][:, :nd], lmask[fixed_rows], dim=0)
                    dx = com_denoised - com_noised
                    z_known[:, :nd] = z_known[:, :nd] + dx[lmask]
                    xh_pocket[:, :nd] = xh_pocket[:, :nd] + dx[pmask]

                    z_lig = z_known * lig_fixed + z_unknown * (1 - lig_fixed)
                    if u < resamplings - 1:
                        z_lig, xh_pocket = self.sample_p_zt_given_zs(z_lig, xh_pocket, lmask, pmask, gamma_t, gamma_s)
                    if u == resamplings - 1 and (s * return_frames) % timesteps == 0:
                        idx = (s * return_frames) // timesteps
                        out_lig[idx], out_pocket[idx] = self.unnormalize_z(z_lig, xh_pocket)

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
    def diversify(self, ligand, pocket, noising_steps):
        """conditional_model.py:364-409: partially noise given ligands, then denoise them again."""
        ligand, pocket = self.normalize(ligand, pocket)
        z_lig, xh_pocket, _ = self.partially_noised_ligand(ligand, pocket, noising_steps)
        timesteps = self.T
        n_samples = len(pocket['size'])
        lig_mask = ligand['mask']
        self.assert_mean_zero_with_mask(z_lig[:, :self.n_dims], lig_mask)
        if self._use_graph(z_lig.device) and noising_steps > 0:
            z_lig, xh_pocket = self._graphed_reverse_steps(z_lig, xh_pocket, lig_mask, pocket['mask'], n_samples,
                                                           noising_steps - 1, noising_steps, timesteps)
        else:
            for s in reversed(range(0, noising_steps)):
                s_array = torch.full((n_samples, 1), fill_value=s, device=z_lig.device)
                t_array = (s_array + 1) / timesteps
                s_array = s_array / timesteps
                z_lig, xh_pocket = self.sample_p_zs_given_zt(s_array, t_array, z_lig.detach(), xh_pocket.detach(),
                                                             lig_mask, pocket['mask'])
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

    @follows_dynamics_determinism
    def forward(self, ligand, pocket, return_info=False):
        """conditional_model.py:727-735: the likelihood is evaluated in the frame of the pocket's centre of mass."""
        pocket_com = scatter_mean(pocket['x'], pocket['mask'], dim=0)
        ligand['x'] = ligand['x'] - pocket_com[ligand['mask']]
        pocket['x'] = pocket['x'] - pocket_com[pocket['mask']]
        return super().forward(ligand, pocket, return_info)

    @follows_dynamics_determinism
    @torch.no_grad()
    def sample_given_pocket(self, pocket, num_nodes_lig, return_frames=1, timesteps=None):
        pocket_com = scatter_mean(pocket['x'], pocket['mask'], dim=0)
        pocket['x'] = pocket['x'] - pocket_com[pocket['mask']]
        return super().sample_given_pocket(pocket, num_nodes_lig, return_frames, timesteps)
