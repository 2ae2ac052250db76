"""Sampling-side members of the reference's ``EnVariationalDiffusion`` (joint ligand+pocket DDPM).

reference: equivariant_diffusion/en_diffusion.py.  Only what the sampling path needs is built: noise
schedule (:1105-1190), alpha/sigma helpers (:83-107, :865-878), (un)normalisation (:880-912), COM helpers
(:919-930), node-count prior (:958-1000), ``sample_p_zs_given_zt`` (:503-557), ``sample_p_xh_given_z0``
(:263-288), ``sample`` (:581-651), and the eval-mode likelihood ``forward`` (:336-469) with its helpers (``kl_prior_with_pocket``,
``log_pxh_given_z0_without_constants``, ``log_constants_p_x_given_z0``, ``gaussian_KL``, ``log_pN``, ``delta_log_px``).
Training (``forward`` in train mode, autograd) raises NotImplementedError.

Class and attribute names are the reference's, so ``LigandPocketDDPM.generate_ligands``'s exact-type
dispatch (lightning_modules.py:814, :837) and Lightning checkpoints (keys ``ddpm.gamma.gamma``,
``ddpm.buffer``, ``ddpm.dynamics.*``) keep working.
"""
from __future__ import annotations

import contextlib
import functools
import math
import threading
from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn


# ---- torch-scatter stand-ins (README.md:60 pins torch-scatter 2.0.9; semantics: output length
# index.max()+1 unless dim_size, mean = sum / count.clamp(min=1)) ------------------------------------
# On CUDA, index_add_ accumulates with floating-point atomics in a timing-dependent order.  Inside
# deterministic_reductions(True) — entered by the DDPM wrappers when their dynamics runs in deterministic mode — a CUDA
# scatter is a segment reduction with a fixed summation order instead: rows are put in index order by a stable sort (a
# no-op permutation for a batch mask, which is non-decreasing; the joint model also scatters two concatenated masks).
# CPU tensors always take the index_add_ path.
_REDUCTIONS = threading.local()


@contextlib.contextmanager
def deterministic_reductions(enabled=True):
    prev = getattr(_REDUCTIONS, 'deterministic', False)
    _REDUCTIONS.deterministic = bool(enabled)
    try:
        yield
    finally:
        _REDUCTIONS.deterministic = prev


def follows_dynamics_determinism(fn):
    """Runs a DDPM method inside deterministic_reductions(dynamics.deterministic_active)."""
    @functools.wraps(fn)
    def wrapper(self, *args, **kwargs):
        dyn = getattr(self, 'dynamics', None)
        if dyn is None:
            dyn = getattr(getattr(self, 'ddpm', None), 'dynamics', None)
        with deterministic_reductions(bool(getattr(dyn, 'deterministic_active', False))):
            return fn(self, *args, **kwargs)
    return wrapper


def _ordered_segments(src, index):
    return src.is_cuda and getattr(_REDUCTIONS, 'deterministic', False)


def scatter_add(src, index, dim=0, dim_size=None):
    assert dim == 0
    n = (int(index.max()) + 1 if index.numel() else 0) if dim_size is None else dim_size
    if _ordered_segments(src, index):
        order = torch.argsort(index, stable=True)
        lengths = torch.bincount(index, minlength=n)[:n]
        return torch.segment_reduce(src[order], 'sum', lengths=lengths, axis=0, unsafe=True)
    out = torch.zeros((n,) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    return out.index_add_(0, index, src)


def scatter_mean(src, index, dim=0, dim_size=None):
    tot = scatter_add(src, index, dim, dim_size)
    if _ordered_segments(src, index):
        cnt = torch.bincount(index, minlength=tot.shape[0])[:tot.shape[0]].to(src.dtype)
        return tot / cnt.clamp(min=1).view((-1,) + (1,) * (tot.dim() - 1))
    cnt = torch.zeros(tot.shape[0], dtype=src.dtype, device=src.device)
    cnt.index_add_(0, index, torch.ones(index.shape[0], dtype=src.dtype, device=src.device))
    return tot / cnt.clamp(min=1).view((-1,) + (1,) * (tot.dim() - 1))


def num_nodes_to_batch_mask(n_samples, num_nodes, device):
    """reference utils.py:146-154."""
    assert isinstance(num_nodes, int) or len(num_nodes) == n_samples
    if isinstance(num_nodes, torch.Tensor):
        num_nodes = num_nodes.to(device)
    return torch.repeat_interleave(torch.arange(n_samples, device=device), num_nodes)


# ---- noise schedules ---------------------------------------------------------------------------------------
def _clip_alpha_ratio(alphas2, floor=0.001):
    """en_diffusion.py:1125-1138: bound alpha_t^2 / alpha_{t-1}^2 from below for sampling stability."""
    ext = np.concatenate([np.ones(1), alphas2])
    ratio = np.clip(ext[1:] / ext[:-1], a_min=floor, a_max=1.0)
    return np.cumprod(ratio)


def polynomial_alphas2(timesteps: int, s: float, power: float):
    """en_diffusion.py:1141-1155: alpha^2 = (1 - (x/steps)^power)^2, ratio-clipped, squeezed to [s, 1-s]."""
    steps = timesteps + 1
    grid = np.linspace(0, steps, steps)
    a2 = _clip_alpha_ratio((1.0 - np.power(grid / steps, power)) ** 2)
    return (1.0 - 2.0 * s) * a2 + s


def cosine_alphas2(timesteps: int, s: float = 0.008):
    """en_diffusion.py:1105-1122 (Nichol & Dhariwal cosine schedule)."""
    steps = timesteps + 2
    grid = np.linspace(0, steps, steps)
    cum = np.cos(((grid / steps) + s) / (1 + s) * np.pi * 0.5) ** 2
    cum = cum / cum[0]
    betas = np.clip(1.0 - cum[1:] / cum[:-1], a_min=0, a_max=0.999)
    return np.cumprod(1.0 - betas)


# ---- few-step samplers (DESIGN §13) --------------------------------------------------------------------------------------
SAMPLERS = ('ddpm', 'ddim', 'dpmpp_2m', 'dpmpp_3m')
MULTISTEP = ('dpmpp_2m', 'dpmpp_3m')          # the samplers that keep x0_hat of earlier steps (DESIGN §13, §15)


def check_sampler(sampler, eta):
    """Raises ValueError unless ``sampler`` is one of SAMPLERS, eta lies in [0, 1], and eta is 0 for every sampler but 'ddim'."""
    if sampler not in SAMPLERS:
        raise ValueError(f"unknown sampler {sampler!r}: expected one of {', '.join(SAMPLERS)}")
    if not 0.0 <= float(eta) <= 1.0:
        raise ValueError(f'eta must lie in [0, 1], got {eta}')
    if float(eta) != 0.0 and sampler != 'ddim':
        raise ValueError(f"eta = {eta} needs sampler='ddim' ({sampler!r} is deterministic)")


def _phi_remainder(h):
    """(e^-h - 1 + h) / h^2 - 1/2 in float64 without the cancellation of the difference: below h = 1/4 its Taylor series
    sum_{j >= 1} (-h)^j / (j + 2)!, summed by Horner to j = 16 (the remainder is below 1e-25 there)."""
    series = torch.zeros_like(h)
    for j in range(16, 0, -1):
        series = (series + 1.0 / math.factorial(j + 2)) * (-h)
    direct = (torch.expm1(-h) + h) / (h * h) - 0.5
    return torch.where(h < 0.25, series, direct)


def fast_coefficients(gamma_s, gamma_t, sampler, eta=0.0):
    """float64 per-step coefficients of the 'ddim', 'dpmpp_2m' and 'dpmpp_3m' steps from gamma at s and t ([N, 1] each, row k = step
    s = k, so that row k + 1 is the step run just before row k).  With alpha^2 = sigmoid(-gamma), sigma^2 = sigmoid(gamma):

    'ddim'     (alpha_{t|s}, alpha_s sigma_t / alpha_t - sqrt(sigma_s^2 - eta^2 st^2), eta st), st = sigma_{t|s} sigma_s / sigma_t:
               the (c0, c1, c2) of z / c0 - c1 eps_hat + c2 noise.  c1 is evaluated as (sigma^2_{t|s} / alpha^2_{t|s} +
               eta^2 st^2) / (sigma_t / alpha_{t|s} + sqrt(sigma_s^2 - eta^2 st^2)), the same number without the cancellation
               of the difference, so that at eta = 1 it is the ancestral sigma^2_{t|s} / (alpha_{t|s} sigma_t) to rounding.
    'dpmpp_2m' (sigma_s / sigma_t, -alpha_s (e^-h - 1), 1 / alpha_t, sigma_t, w), h = lambda_s - lambda_t, lambda = -gamma / 2,
               w = h / (2 h_prev) with h_prev the h of row k + 1, and w = 0 in the last row (the first step run).
    'dpmpp_3m' (sigma_s / sigma_t, 1 / alpha_t, sigma_t, k0, k1, k2): z_s = c0 z_t + k0 m0 + k1 m1 + k2 m2 with m0 = x0_hat of
               this step and m1, m2 those of the two steps run before it (DESIGN §15).  The first step run (last row) is
               DDIM at eta = 0 (k0 = -alpha_s phi1, phi1 = e^-h - 1), the second is 2M's second step (k0 = -alpha_s phi1
               (1 + w), k1 = alpha_s phi1 w), every later one third order: with h1, h2 the h of rows k + 1, k + 2,
               D1 = D1_0 + h1 / (h1 + h2) (D1_0 - D1_1), D2 = h (D1_0 - D1_1) / (h1 + h2), D1_0 = h (m0 - m1) / h1,
               D1_1 = h (m1 - m2) / h2, z_s = c0 z_t - alpha_s phi1 m0 + alpha_s (phi1 / h + 1) D1 - alpha_s ((phi1 + h) / h^2
               - 1/2) D2, collected per m.  phi1 / h + 1 = h (g + 1/2) and (phi1 + h) / h^2 - 1/2 = g come from
               _phi_remainder, so no difference cancels at small h; every k is then a sum of same-signed terms."""
    gs, gt = gamma_s.detach().double(), gamma_t.detach().double()
    s2_s, s2_t = torch.sigmoid(gs), torch.sigmoid(gt)
    alpha_s, alpha_t = torch.sqrt(torch.sigmoid(-gs)), torch.sqrt(torch.sigmoid(-gt))
    sigma_s, sigma_t = torch.sqrt(s2_s), torch.sqrt(s2_t)
    if sampler == 'ddim':
        eta2 = float(eta) ** 2
        sigma2_ts = -torch.expm1(F.softplus(gs) - F.softplus(gt))
        alpha_ts = torch.exp(0.5 * (F.logsigmoid(-gt) - F.logsigmoid(-gs)))
        tilde2 = sigma2_ts * s2_s / s2_t
        # sigma_s^2 - eta^2 tilde^2 = sigma_s^2 (alpha_ts^2 sigma_s^2 + (1 - eta^2) sigma2_ts) / sigma_t^2, a sum of non-negatives
        keep = torch.sqrt(s2_s * (alpha_ts ** 2 * s2_s + (1.0 - eta2) * sigma2_ts) / s2_t)
        c1 = (sigma2_ts / alpha_ts ** 2 + eta2 * tilde2) / (sigma_t / alpha_ts + keep)
        return torch.cat([alpha_ts, c1, float(eta) * torch.sqrt(tilde2)], dim=1)
    if sampler == 'dpmpp_2m':
        h = 0.5 * (gt - gs)
        w = torch.zeros_like(h)
        w[:-1] = h[:-1] / (2.0 * h[1:])
        return torch.cat([sigma_s / sigma_t, -alpha_s * torch.expm1(-h), 1.0 / alpha_t, sigma_t, w], dim=1)
    if sampler == 'dpmpp_3m':
        h = 0.5 * (gt - gs)
        c1 = -alpha_s * torch.expm1(-h)
        g = _phi_remainder(h)
        k = torch.zeros((h.shape[0], 3), dtype=h.dtype, device=h.device)
        k[-1:, 0:1] = c1[-1:]                                       # first step run: order 1
        if h.shape[0] >= 2:                                          # second: order 2, as 2M
            w = h[-2:-1] / (2.0 * h[-1:])
            k[-2:-1, 0:1], k[-2:-1, 1:2] = c1[-2:-1] * (1.0 + w), -c1[-2:-1] * w
        if h.shape[0] >= 3:                                          # the rest: order 3
            hh, h1, h2, a_s = h[:-2], h[1:-1], h[2:], alpha_s[:-2]
            A, B = a_s * hh * (g[:-2] + 0.5), -a_s * g[:-2]          # alpha_s (phi1 / h + 1), -alpha_s ((phi1 + h) / h^2 - 1/2)
            a0 = A * (1.0 + h1 / (h1 + h2)) + B * hh / (h1 + h2)     # the weights of D1_0 and D1_1
            a1 = -A * h1 / (h1 + h2) - B * hh / (h1 + h2)
            k[:-2] = torch.cat([c1[:-2] + a0 * hh / h1, -a0 * hh / h1 + a1 * hh / h2, -a1 * hh / h2], dim=1)
        return torch.cat([sigma_s / sigma_t, 1.0 / alpha_t, sigma_t, k], dim=1)
    raise ValueError(sampler)


def multistep_update(z, eps, hist, c):
    """The 'dpmpp_2m' / 'dpmpp_3m' update of one part, rows of ``c`` per node (fast_coefficients), before its COM removal.
    ``hist``: the x0_hat of the steps run before, newest first: (m1,) for 2M, (m1, m2) for 3M.  Returns (z', the history a
    commit writes): (x0_hat,) for 2M; (x0_hat, m2') for 3M, where m2' = m1, or x0_hat on the first step run (k1 = 0)."""
    if len(hist) == 1:
        x0 = (z - c[:, 3:4] * eps) * c[:, 2:3]
        return c[:, 0:1] * z + c[:, 1:2] * ((1 + c[:, 4:5]) * x0 - c[:, 4:5] * hist[0]), (x0,)
    m1, m2 = hist
    x0 = (z - c[:, 2:3] * eps) * c[:, 1:2]
    out = c[:, 0:1] * z + c[:, 3:4] * x0 + c[:, 4:5] * m1 + c[:, 5:6] * m2
    return out, (x0, torch.where(c[:, 4:5] != 0, m1, x0))


class PredefinedNoiseSchedule(nn.Module):
    """Lookup table gamma[t_int] = -(log alpha^2 - log sigma^2) (en_diffusion.py:1158-1190)."""

    def __init__(self, noise_schedule, timesteps, precision):
        super().__init__()
        self.timesteps = timesteps
        if noise_schedule == 'cosine':
            a2 = cosine_alphas2(timesteps)
        elif 'polynomial' in noise_schedule:
            parts = noise_schedule.split('_')
            assert len(parts) == 2
            a2 = polynomial_alphas2(timesteps, s=precision, power=float(parts[1]))
        else:
            raise ValueError(noise_schedule)
        log_ratio = np.log(a2) - np.log(1.0 - a2)
        self.gamma = nn.Parameter(torch.from_numpy(-log_ratio).float(), requires_grad=False)

    def forward(self, t):
        return self.gamma[torch.round(t * self.timesteps).long()]


class PositiveLinear(nn.Module):
    """Linear layer with softplus-positive weights (en_diffusion.py:1031-1061); kept so checkpoints with a
    learned schedule restore (``ddpm.gamma.l{1,2,3}.*``)."""

    def __init__(self, in_features, out_features, bias=True, weight_init_offset=-2):
        super().__init__()
        self.weight = nn.Parameter(torch.empty((out_features, in_features)))
        self.bias = nn.Parameter(torch.empty(out_features)) if bias else None
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        with torch.no_grad():
            self.weight.add_(weight_init_offset)
        if bias:
            bound = 1.0 / math.sqrt(in_features) if in_features > 0 else 0
            nn.init.uniform_(self.bias, -bound, bound)

    def forward(self, x):
        return F.linear(x, F.softplus(self.weight), self.bias)


class GammaNetwork(nn.Module):
    """Monotone learned gamma(t) (en_diffusion.py:1064-1102)."""

    def __init__(self):
        super().__init__()
        self.l1, self.l2, self.l3 = PositiveLinear(1, 1), PositiveLinear(1, 1024), PositiveLinear(1024, 1)
        self.gamma_0 = nn.Parameter(torch.tensor([-5.]))
        self.gamma_1 = nn.Parameter(torch.tensor([10.]))

    def _tilde(self, t):
        a = self.l1(t)
        return a + self.l3(torch.sigmoid(self.l2(a)))

    def forward(self, t):
        g0, g1, gt = self._tilde(torch.zeros_like(t)), self._tilde(torch.ones_like(t)), self._tilde(t)
        return self.gamma_0 + (self.gamma_1 - self.gamma_0) * (gt - g0) / (g1 - g0)


class DistributionNodes:
    """Joint histogram over (ligand size, pocket size); en_diffusion.py:958-1028 (sampling members)."""

    def __init__(self, histogram):
        hist = torch.tensor(histogram).float() + 1e-3
        self.prob = hist / hist.sum()
        n1, n2 = self.prob.shape
        self.idx_to_n_nodes = torch.stack(torch.meshgrid(torch.arange(n1), torch.arange(n2), indexing='ij'),
                                          dim=-1).view(-1, 2)
        self.n_nodes_to_idx = {tuple(v.tolist()): i for i, v in enumerate(self.idx_to_n_nodes)}
        self.m = torch.distributions.Categorical(self.prob.view(-1), validate_args=True)
        self.n1_given_n2 = [torch.distributions.Categorical(self.prob[:, j], validate_args=True) for j in range(n2)]
        self.n2_given_n1 = [torch.distributions.Categorical(self.prob[i, :], validate_args=True) for i in range(n1)]

    def sample(self, n_samples=1):
        lig, pocket = self.idx_to_n_nodes[self.m.sample((n_samples,))].T
        return lig, pocket

    def sample_conditional(self, n1=None, n2=None):
        assert (n1 is None) ^ (n2 is None), "Exactly one input argument must be None"
        dists, cond = (self.n1_given_n2, n2) if n2 is not None else (self.n2_given_n1, n1)
        return torch.tensor([dists[int(i)].sample() for i in cond], device=cond.device)

    def log_prob(self, batch_n_nodes_1, batch_n_nodes_2):
        """en_diffusion.py:1002-1014: log p(n_ligand, n_pocket) under the joint histogram."""
        assert batch_n_nodes_1.dim() == 1 and batch_n_nodes_2.dim() == 1
        idx = torch.tensor([self.n_nodes_to_idx[pair] for pair in zip(batch_n_nodes_1.tolist(), batch_n_nodes_2.tolist())])
        return self.m.log_prob(idx).to(batch_n_nodes_1.device)

    def log_prob_n1_given_n2(self, n1, n2):
        return torch.stack([self.n1_given_n2[int(c)].log_prob(i.cpu()) for i, c in zip(n1, n2)]).to(n1.device)


class EnVariationalDiffusion(nn.Module):
    """reference en_diffusion.py:13 (constructor :18-66).

    ``loop_engine``: 'auto' | 'graph' | 'eager'.  On CUDA with the native denoiser, ``sample`` and ``inpaint`` replay
    captured CUDA graphs (denoiser + fused joint update / RePaint iteration, libdiffsbdd_b200 ``dsb_ddpm_joint_update`` /
    ``dsb_ddpm_joint_inpaint_update``); 'eager' keeps the reference-order Python loop (same torch ops, same RNG calls)."""

    loop_engine = 'auto'
    _rng = None              # seeded.SeededDraws of the running seeded sampler call (None: torch's global generator)

    def __init__(self, dynamics: nn.Module, atom_nf: int, residue_nf: int, n_dims: int, size_histogram: Dict,
                 timesteps: int = 1000, parametrization='eps', noise_schedule='learned', noise_precision=1e-4,
                 loss_type='vlb', norm_values=(1., 1.), norm_biases=(None, 0.), virtual_node_idx=None):
        super().__init__()
        assert loss_type in {'vlb', 'l2'}
        assert parametrization == 'eps'
        self.loss_type = loss_type
        if noise_schedule == 'learned':
            assert loss_type == 'vlb', 'A noise schedule can only be learned with a vlb objective.'
            self.gamma = GammaNetwork()
        else:
            self.gamma = PredefinedNoiseSchedule(noise_schedule, timesteps=timesteps, precision=noise_precision)
        self.dynamics = dynamics
        self.atom_nf, self.residue_nf, self.n_dims = atom_nf, residue_nf, n_dims
        self.num_classes = atom_nf
        self.T = timesteps
        self.parametrization = parametrization
        self.norm_values, self.norm_biases = norm_values, norm_biases
        self.register_buffer('buffer', torch.zeros(1))
        self.size_distribution = DistributionNodes(size_histogram)
        self.vnode_idx = virtual_node_idx
        self._joint_cache = {}                 # captured CUDA graphs of the joint samplers (see _joint_engine)
        if noise_schedule != 'learned':
            self.check_issues_norm_values()

    # ---- schedule algebra (en_diffusion.py:68-107, :865-878) ---------------------------------------------
    def check_issues_norm_values(self, num_stdevs=8):
        zeros = torch.zeros((1, 1))
        sigma_0 = self.sigma(self.gamma(zeros), target_tensor=zeros).item()
        if sigma_0 * num_stdevs > 1. / self.norm_values[1]:
            raise ValueError(f'Value for normalization value {self.norm_values[1]} probably too large with '
                             f'sigma_0 {sigma_0:.5f} and 1 / norm_value = {1. / self.norm_values[1]}')

    @staticmethod
    def inflate_batch_array(array, target):
        return array.view((array.size(0),) + (1,) * (len(target.size()) - 1))

    def sigma(self, gamma, target_tensor):
        return self.inflate_batch_array(torch.sqrt(torch.sigmoid(gamma)), target_tensor)

    def alpha(self, gamma, target_tensor):
        return self.inflate_batch_array(torch.sqrt(torch.sigmoid(-gamma)), target_tensor)

    @staticmethod
    def SNR(gamma):
        return torch.exp(-gamma)

    def sigma_and_alpha_t_given_s(self, gamma_t, gamma_s, target_tensor):
        sigma2 = self.inflate_batch_array(-torch.expm1(F.softplus(gamma_s) - F.softplus(gamma_t)), target_tensor)
        log_a2 = F.logsigmoid(-gamma_t) - F.logsigmoid(-gamma_s)
        alpha = self.inflate_batch_array(torch.exp(0.5 * log_a2), target_tensor)
        return sigma2, torch.sqrt(sigma2), alpha

    # ---- data scaling (en_diffusion.py:880-912) ------------------------------------------------------------
    def normalize(self, ligand=None, pocket=None):
        for part in (ligand, pocket):
            if part is not None:
                part['x'] = part['x'] / self.norm_values[0]
                part['one_hot'] = (part['one_hot'].float() - self.norm_biases[1]) / self.norm_values[1]
        return ligand, pocket

    def unnormalize(self, x, h_cat):
        return x * self.norm_values[0], h_cat * self.norm_values[1] + self.norm_biases[1]

    def unnormalize_z(self, z_lig, z_pocket):
        nd = self.n_dims
        xl, hl = self.unnormalize(z_lig[:, :nd], z_lig[:, nd:])
        xp, hp = self.unnormalize(z_pocket[:, :nd], z_pocket[:, nd:])
        return torch.cat([xl, hl], dim=1), torch.cat([xp, hp], dim=1)

    def subspace_dimensionality(self, input_size):
        return (input_size - 1) * self.n_dims

    # ---- COM helpers (en_diffusion.py:919-955) -------------------------------------------------------------
    @staticmethod
    def remove_mean_batch(x, indices):
        return x - scatter_mean(x, indices, dim=0)[indices]

    @staticmethod
    def assert_mean_zero_with_mask(x, node_mask, eps=1e-10):
        largest = x.abs().max().item()
        error = scatter_add(x, node_mask, dim=0).abs().max().item()
        rel = error / (largest + eps)
        assert rel < 1e-2, f'Mean is not zero, relative_error {rel}'

    @staticmethod
    def sample_center_gravity_zero_gaussian_batch(size, lig_indices, pocket_indices):
        assert len(size) == 2
        x = torch.randn(size, device=lig_indices.device)
        return EnVariationalDiffusion.remove_mean_batch(x, torch.cat((lig_indices, pocket_indices)))

    @staticmethod
    def sample_gaussian(size, device):
        return torch.randn(size, device=device)

    # ---- seeded draws (seeded.py): active inside a sampler call that was given seeds= -----------------------------
    @contextlib.contextmanager
    def _seeded(self, seeds, lig_mask, pocket_mask):
        from .seeded import SeededDraws
        prev = self._rng
        self._rng = None if seeds is None else SeededDraws(seeds, lig_mask, pocket_mask)
        try:
            yield
        finally:
            self._rng = prev

    def _draw_at(self, stage, s=0, u=0, purpose=0):
        """Sets the draw id of the next seeded draws (no-op without seeds)."""
        if self._rng is not None:
            self._rng.at(stage, s, u, purpose)

    def _seeds(self):
        return None if self._rng is None else self._rng.seeds

    def _lig_noise(self, lig_mask, cols):
        if self._rng is None:
            return self.sample_gaussian(size=(len(lig_mask), cols), device=lig_mask.device)
        from ._native import RNG_LIGAND
        return self._rng.normal(RNG_LIGAND, cols)

    def _project_cog_drift(self, x_lig, x_pocket, lig_mask, project, pocket_mask, x_all=None, all_mask=None):
        """The final CoG-drift projection of the samplers (conditional_model.py:540-547, en_diffusion.py:637-646): without
        seeds, as the reference, every graph is projected when any graph's CoG exceeds 5e-2.  With seeds only the graphs whose
        own CoG exceeds it are projected, so that a graph's result does not depend on its batch (the one deviation from the
        reference, and only with seeds).  ``project()`` returns the projected (x_lig, x_pocket)."""
        cog = scatter_add(x_lig if x_all is None else x_all, lig_mask if all_mask is None else all_mask, dim=0).abs()
        if self._rng is None:
            max_cog = cog.max().item()
            if max_cog > 5e-2:
                print(f'Warning CoG drift with error {max_cog:.3f}. Projecting the positions down.')
                return project()
            return x_lig, x_pocket
        drift = cog.amax(dim=1) > 5e-2
        if not bool(drift.any()):
            return x_lig, x_pocket
        print(f'Warning CoG drift in {int(drift.sum())} graph(s), max error {cog.max().item():.3f}. Projecting those graphs.')
        pl, pp = project()
        return (torch.where(drift[lig_mask].unsqueeze(1), pl, x_lig), torch.where(drift[pocket_mask].unsqueeze(1), pp, x_pocket))

    @staticmethod
    def sum_except_batch(x, indices):
        return scatter_add(x.sum(-1), indices, dim=0)

    def compute_x_pred(self, net_out, zt, gamma_t, batch_mask):
        """en_diffusion.py:157-169 (eps parametrisation)."""
        sigma_t = self.sigma(gamma_t, target_tensor=net_out)
        alpha_t = self.alpha(gamma_t, target_tensor=net_out)
        return 1. / alpha_t[batch_mask] * (zt - sigma_t[batch_mask] * net_out)

    def xh_given_zt_and_epsilon(self, z_t, epsilon, gamma_t, batch_mask):
        alpha_t, sigma_t = self.alpha(gamma_t, z_t), self.sigma(gamma_t, z_t)
        return z_t / alpha_t[batch_mask] - epsilon * sigma_t[batch_mask] / alpha_t[batch_mask]

    # ---- joint sampling (en_diffusion.py:263-301, :503-651) -----------------------------------------------
    def sample_combined_position_feature_noise(self, lig_indices, pocket_indices):
        """en_diffusion.py:559-578: COM-free x noise over ligand+pocket, plain h noise."""
        nl, npk = len(lig_indices), len(pocket_indices)
        if self._rng is not None:
            from . import _native
            zx = self.remove_mean_batch(self._rng.normal(_native.RNG_JOINT_X, self.n_dims), torch.cat((lig_indices, pocket_indices)))
            return (torch.cat([zx[:nl], self._rng.normal(_native.RNG_LIGAND, self.atom_nf)], dim=1),
                    torch.cat([zx[nl:], self._rng.normal(_native.RNG_POCKET, self.residue_nf)], dim=1))
        zx = self.sample_center_gravity_zero_gaussian_batch((nl + npk, self.n_dims), lig_indices, pocket_indices)
        z_lig = torch.cat([zx[:nl], self.sample_gaussian((nl, self.atom_nf), lig_indices.device)], dim=1)
        z_pocket = torch.cat([zx[nl:], self.sample_gaussian((npk, self.residue_nf), pocket_indices.device)], dim=1)
        return z_lig, z_pocket

    def sample_normal(self, mu_lig, mu_pocket, sigma, lig_mask, pocket_mask, fix_noise=False):
        if fix_noise:
            raise NotImplementedError("fix_noise option isn't implemented yet")
        eps_lig, eps_pocket = self.sample_combined_position_feature_noise(lig_mask, pocket_mask)
        return mu_lig + sigma[lig_mask] * eps_lig, mu_pocket + sigma[pocket_mask] * eps_pocket

    def noised_representation(self, xh_lig, xh_pocket, lig_mask, pocket_mask, gamma_t):
        """en_diffusion.py:302-317: z_t ~ q(z_t | x, h) for ligand and pocket."""
        alpha_t, sigma_t = self.alpha(gamma_t, xh_lig), self.sigma(gamma_t, xh_lig)
        eps_lig, eps_pocket = self.sample_combined_position_feature_noise(lig_mask, pocket_mask)
        z_lig = alpha_t[lig_mask] * xh_lig + sigma_t[lig_mask] * eps_lig
        z_pocket = alpha_t[pocket_mask] * xh_pocket + sigma_t[pocket_mask] * eps_pocket
        return z_lig, z_pocket, eps_lig, eps_pocket

    def _project_joint_com(self, z_lig, z_pocket, ligand_mask, pocket_mask):
        nl = len(ligand_mask)
        zx = self.remove_mean_batch(torch.cat((z_lig[:, :self.n_dims], z_pocket[:, :self.n_dims]), dim=0),
                                    torch.cat((ligand_mask, pocket_mask)))
        return (torch.cat((zx[:nl], z_lig[:, self.n_dims:]), dim=1),
                torch.cat((zx[nl:], z_pocket[:, self.n_dims:]), dim=1))

    def sample_p_zt_given_zs(self, zs_lig, zs_pocket, ligand_mask, pocket_mask, gamma_t, gamma_s, fix_noise=False):
        """en_diffusion.py:479-501: forward (re-noising) step used by RePaint."""
        _, sigma_ts, alpha_ts = self.sigma_and_alpha_t_given_s(gamma_t, gamma_s, zs_lig)
        zt_lig, zt_pocket = self.sample_normal(alpha_ts[ligand_mask] * zs_lig, alpha_ts[pocket_mask] * zs_pocket,
                                               sigma_ts, ligand_mask, pocket_mask, fix_noise)
        return self._project_joint_com(zt_lig, zt_pocket, ligand_mask, pocket_mask)

    def sample_p_zs_given_zt(self, s, t, zt_lig, zt_pocket, ligand_mask, pocket_mask, fix_noise=False):
        """en_diffusion.py:503-557: joint reverse step; the x-mean of the combined system is projected out."""
        gamma_s, gamma_t = self.gamma(s), self.gamma(t)
        sigma2_ts, sigma_ts, alpha_ts = self.sigma_and_alpha_t_given_s(gamma_t, gamma_s, zt_lig)
        sigma_s = self.sigma(gamma_s, target_tensor=zt_lig)
        sigma_t = self.sigma(gamma_t, target_tensor=zt_lig)
        eps_lig, eps_pocket = self.dynamics(zt_lig, zt_pocket, t, ligand_mask, pocket_mask)
        combined_mask = torch.cat((ligand_mask, pocket_mask))
        self.assert_mean_zero_with_mask(
            torch.cat((zt_lig[:, :self.n_dims], zt_pocket[:, :self.n_dims]), dim=0), combined_mask)
        self.assert_mean_zero_with_mask(
            torch.cat((eps_lig[:, :self.n_dims], eps_pocket[:, :self.n_dims]), dim=0), combined_mask)
        coef = sigma2_ts / alpha_ts / sigma_t
        mu_lig = zt_lig / alpha_ts[ligand_mask] - coef[ligand_mask] * eps_lig
        mu_pocket = zt_pocket / alpha_ts[pocket_mask] - coef[pocket_mask] * eps_pocket
        sigma = sigma_ts * sigma_s / sigma_t
        zs_lig, zs_pocket = self.sample_normal(mu_lig, mu_pocket, sigma, ligand_mask, pocket_mask, fix_noise)
        return self._project_joint_com(zs_lig, zs_pocket, ligand_mask, pocket_mask)

    def sample_p_xh_given_z0(self, z0_lig, z0_pocket, lig_mask, pocket_mask, batch_size, fix_noise=False):
        """en_diffusion.py:263-288."""
        t_zeros = torch.zeros(size=(batch_size, 1), device=z0_lig.device)
        gamma_0 = self.gamma(t_zeros)
        sigma_x = self.SNR(-0.5 * gamma_0)
        out_lig, out_pocket = self.dynamics(z0_lig, z0_pocket, t_zeros, lig_mask, pocket_mask)
        mu_lig = self.compute_x_pred(out_lig, z0_lig, gamma_0, lig_mask)
        mu_pocket = self.compute_x_pred(out_pocket, z0_pocket, gamma_0, pocket_mask)
        xh_lig, xh_pocket = self.sample_normal(mu_lig, mu_pocket, sigma_x, lig_mask, pocket_mask, fix_noise)
        x_lig, h_lig = self.unnormalize(xh_lig[:, :self.n_dims], z0_lig[:, self.n_dims:])
        x_pocket, h_pocket = self.unnormalize(xh_pocket[:, :self.n_dims], z0_pocket[:, self.n_dims:])
        h_lig = F.one_hot(torch.argmax(h_lig, dim=1), self.atom_nf)
        h_pocket = F.one_hot(torch.argmax(h_pocket, dim=1), self.residue_nf)
        return x_lig, h_lig, x_pocket, h_pocket

    # ---- CUDA-graphed joint loops (SURVEY.md §8 f3) ---------------------------------------------------------------
    def _joint_use_graph(self, device) -> bool:
        from .dynamics import EGNNDynamics
        if self.loop_engine == 'eager' or type(self) is not EnVariationalDiffusion:
            return False
        ok = isinstance(self.dynamics, EGNNDynamics) and torch.device(device).type == 'cuda'
        if self.loop_engine == 'graph' and not ok:
            raise RuntimeError("loop_engine='graph' needs the native EGNNDynamics on a CUDA device")
        return ok

    def _joint_tables(self, timesteps, jump_length, device):
        """Per-step scalars (s = 0..timesteps-1, t = s+1) from the same fp32 torch ops as the eager steps:
        t | reverse (alpha_{t|s}, sigma^2_{t|s}/alpha_{t|s}/sigma_t, sigma_{t|s} sigma_s/sigma_t) |
        RePaint (alpha_s, sigma_s, alpha_{s+j|s}, sigma_{s+j|s}) — en_diffusion.py:503-557, :302-317, :479-501."""
        s_int = torch.arange(timesteps, device=device).view(-1, 1)
        t_arr, s_arr = (s_int + 1) / timesteps, s_int / timesteps
        gamma_s, gamma_t = self.gamma(s_arr), self.gamma(t_arr)
        sigma2_ts, sigma_ts, alpha_ts = self.sigma_and_alpha_t_given_s(gamma_t, gamma_s, s_arr)
        sigma_s, sigma_t = self.sigma(gamma_s, s_arr), self.sigma(gamma_t, s_arr)
        rev = [alpha_ts, sigma2_ts / alpha_ts / sigma_t, sigma_ts * sigma_s / sigma_t]
        t_back = torch.clamp(s_int + jump_length, max=timesteps) / timesteps
        _, sig_j, alp_j = self.sigma_and_alpha_t_given_s(self.gamma(t_back), gamma_s, s_arr)
        inp = [self.alpha(gamma_s, s_arr), self.sigma(gamma_s, s_arr), alp_j, sig_j]
        return t_arr.float().contiguous(), torch.cat(rev + inp, dim=1).float().contiguous()

    def _fast_tables(self, timesteps, sampler, eta, device, top=None):
        """Per-step t and coefficients of the 'ddim' / 'dpmpp_2m' / 'dpmpp_3m' steps s = 0..timesteps-1 (t = s+1) for both engines:
        fast_coefficients in float64 from the fp32 gamma values, cast to fp32, so that eager and graph steps use the same bits.
        ``top`` = (n, T): the grid ends at t* = n / T instead of 1 (diversify), t_k = k n / (timesteps T) in one rounding."""
        s_int = torch.arange(timesteps, device=device).view(-1, 1)
        if top is None:
            t_arr, s_arr = (s_int + 1) / timesteps, s_int / timesteps
        else:
            t_arr, s_arr = (s_int + 1) * top[0] / (timesteps * top[1]), s_int * top[0] / (timesteps * top[1])
        coef = fast_coefficients(self.gamma(s_arr), self.gamma(t_arr), sampler, eta)
        return t_arr.float().contiguous(), coef.float().contiguous()

    @staticmethod
    def _eager_row(s, timesteps, n_samples, device, fast):
        """(t, row) of eager step s as _fast_step / _joint_fast_step take them.  'ddpm' (``fast`` None): the reference's
        t = (s + 1) / timesteps and s / timesteps, [n_samples, 1] each; else t and the step's row [1, k] of ``fast``, the
        (t, coefficients) pair of _fast_tables."""
        if fast is None:
            s_array = torch.full((n_samples, 1), fill_value=s, device=device)
            return (s_array + 1) / timesteps, s_array / timesteps
        t_table, coef = fast
        return t_table[s].expand(n_samples, 1), coef[s:s + 1]

    def _joint_engine(self, z_lig, z_pocket, lig_mask, pocket_mask, n_samples, timesteps, jump_length, sampler='ddpm', eta=0.0):
        dyn = self.dynamics
        device = z_lig.device
        dyn._ensure_handle(device)
        seeds = self._seeds()
        key = (tuple(z_lig.shape), tuple(z_pocket.shape), n_samples, timesteps, jump_length, str(device), seeds is not None,
               sampler, eta)
        st = self._joint_cache.get(key)
        if st is not None:
            same = torch.equal(st['lig_mask'], lig_mask) and torch.equal(st['pocket_mask'], pocket_mask)
            if not same or st['sig'] != dyn.capture_signature():
                st = None
        if st is None:
            self._joint_cache.clear()
            t_table, coef_table = self._joint_tables(timesteps, jump_length, device)
            nl, npk = z_lig.shape[0], z_pocket.shape[0]
            noise = lambda: (torch.empty((nl + npk, self.n_dims), device=device), torch.empty((nl, self.atom_nf), device=device),
                             torch.empty((npk, self.residue_nf), device=device))
            st = dict(zl=torch.empty_like(z_lig), zp=torch.empty_like(z_pocket), n_rev=noise(), n_known=noise(), n_jump=noise(),
                      t=torch.zeros((n_samples, 1), device=device), coef3=torch.zeros((n_samples, 3), device=device),
                      coef4=torch.zeros((n_samples, 4), device=device), step=torch.zeros(1, dtype=torch.int64, device=device),
                      t_table=t_table, coef_table=coef_table, lig_mask=lig_mask.clone(), pocket_mask=pocket_mask.clone(),
                      graphs={}, sig=None, n_samples=n_samples, jump=jump_length, known=None, seeded=seeds is not None)
            if seeds is not None:     # seeds, draw ids of the step's three draws, jumps back so far u
                st.update(seeds=torch.empty_like(seeds), draw=torch.zeros(3, dtype=torch.int64, device=device),
                          u=torch.zeros(1, dtype=torch.int64, device=device))
            if sampler != 'ddpm':     # few-step samplers: their coefficient table; DDIM at eta = 0 adds 0 * (zeroed noise)
                _, fast = self._fast_tables(timesteps, sampler, eta, device)
                st.update(fast_table=fast, coef_fast=torch.zeros((n_samples, fast.shape[1]), device=device), eta=eta,
                          sampler=sampler)
                for x in st['n_rev']:
                    x.zero_()
                if sampler in MULTISTEP:   # RePaint rounds: the 2M / 3M row and the RePaint row in one [n, 9 | 10] buffer
                    st['hist'] = (torch.zeros_like(z_lig), torch.zeros_like(z_pocket))
                    if sampler == 'dpmpp_3m':
                        st['hist2'] = (torch.zeros_like(z_lig), torch.zeros_like(z_pocket))
                    ms = torch.cat((fast, coef_table[:, 3:]), 1).contiguous()
                    st['ms_table'] = ms
                    st['coef9' if sampler == 'dpmpp_2m' else 'coef10'] = torch.zeros((n_samples, ms.shape[1]), device=device)
            self._joint_cache[key] = st
        if seeds is not None:
            st['seeds'].copy_(seeds)
            st['u'].zero_()
        return st

    def _joint_step(self, st, kind):
        """One iteration of the joint model as a python callable over the static buffers of ``st``, with the step of the
        sampler the engine was built for.  kind: 'reverse' ('ddpm') | 'ddim' | 'dpmpp_2m' | 'dpmpp_3m' (one joint step,
        step -= 1) | 'inpaint' (noised known part + the step + blend, step -= 1; 2M / 3M: commits its x0_hat as the history) |
        'inpaint_jump' (the same + jump back by jump_length, no commit: step += jump_length - 1, u += 1) | 'inpaint_hold'
        (as 'inpaint' without the commit: a frame is taken before an eager jump back) (DESIGN §13-15).  A run: draw ids ->
        the step's table rows -> native denoiser -> draws -> dsb_ddpm_joint_update (+ dsb_ddpm_joint_inpaint_update), or the
        2M / 3M step or RePaint round (_native.multistep_update) -> counters."""
        import ctypes as C
        from . import _native, seeded
        dyn, lib = self.dynamics, _native.load()
        lm, pm, n = st['lig_mask'], st['pocket_mask'], st['n_samples']
        sizes = (st['zl'].shape[0], st['zp'].shape[0], n, self.atom_nf, self.residue_nf)
        ptr = lambda x: None if x is None else x.data_ptr()
        roles = (_native.RNG_JOINT_X, _native.RNG_LIGAND, _native.RNG_POCKET)
        sampler = st.get('sampler', 'ddpm')
        repaint, jump = kind.startswith('inpaint'), kind == 'inpaint_jump'
        # table rows -> the buffers the kernels read, {table: [(buffer, first column)]}; one index_select per table
        coef = 'coef3' if sampler == 'ddpm' else 'coef_fast'
        if repaint and sampler in MULTISTEP:      # the 2M / 3M row and the RePaint row in one [n, 9 | 10] buffer
            coef = 'coef9' if sampler == 'dpmpp_2m' else 'coef10'
            stage = {'ms_table': [(coef, 0)]}
        else:
            stage = {'coef_table' if sampler == 'ddpm' else 'fast_table': [(coef, 0)]}
            if repaint:                           # the RePaint row of dsb_ddpm_joint_inpaint_update
                stage.setdefault('coef_table', []).append(('coef4', 3))
        # the step's draws in eager order (en_diffusion.py:741): known part, reverse noise ('ddpm', DDIM at eta > 0), jump
        draws = [(p, buf) for p, buf, on in ((seeded.PURPOSE_KNOWN, 'n_known', repaint),
                                             (seeded.PURPOSE_REVERSE, 'n_rev', sampler == 'ddpm' or st.get('eta', 0) > 0),
                                             (seeded.PURPOSE_RENOISE, 'n_jump', jump)) if on]

        def run():
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
            if st['seeded'] and draws:
                seeded.graph_draw_ids(st['step'], st['u'], st['draw'])
            idx = st['step'].clamp(min=0)
            st['t'].copy_(st['t_table'].index_select(0, idx).expand(n, 1))
            for table, bufs in stage.items():
                row = st[table].index_select(0, idx)
                for key, c0 in bufs:
                    st[key].copy_(row[:, c0:c0 + st[key].shape[1]].expand_as(st[key]))
            eps_l, eps_p = dyn(st['zl'], st['zp'], st['t'], lm, pm)
            for p, buf in draws:
                for x, role in zip(st[buf], roles):
                    if st['seeded']:
                        seeded.fill(x, role, st['seeds'], st['draw'][p:p + 1], lm, pm)
                    else:
                        x.normal_()
            kn = st['known']
            n_jump = st['n_jump'] if jump else (None,) * 3
            if sampler in MULTISTEP:
                rp = (kn['xl'], kn['xp'], None, kn['fl'], kn['fp'], *st['n_known'], *n_jump) if repaint else ()
                _native.multistep_update(lib, (st['zl'], st['zp']), self._joint_static_history(st), (eps_l, eps_p), st[coef],
                                         (lm, pm), sizes, 1, stream, rp, int(kind == 'inpaint'))
            else:
                _native.check(lib.dsb_ddpm_joint_update(
                    ptr(st['zl']), ptr(st['zp']), ptr(eps_l), ptr(eps_p), *map(ptr, st['n_rev']), ptr(st[coef]), ptr(lm),
                    ptr(pm), *sizes, stream))
                if repaint:
                    _native.check(lib.dsb_ddpm_joint_inpaint_update(
                        ptr(st['zl']), ptr(st['zp']), ptr(kn['xl']), ptr(kn['xp']), ptr(kn['fl']), ptr(kn['fp']),
                        *map(ptr, st['n_known']), *map(ptr, n_jump), ptr(st['coef4']), ptr(lm), ptr(pm), *sizes, stream))
            if jump:
                st['step'].add_(st['jump'] - 1)
                if st['seeded']:
                    st['u'].add_(1)
            else:
                st['step'].sub_(1)
        return run

    @staticmethod
    def _joint_start(st, z_lig, z_pocket, first_s):
        """Loads the static state a run of captured joint steps starts from: z, step and (seeded) the jump count u = 0.  A
        warm-up run advances u like any other, so capture resets it here as well."""
        st['zl'].copy_(z_lig); st['zp'].copy_(z_pocket); st['step'].fill_(first_s)
        if st['seeded']:
            st['u'].zero_()
        for x in st.get('hist', ()) + st.get('hist2', ()):
            x.zero_()

    @staticmethod
    def _joint_static_history(st):
        """The multistep histories of the static state, newest first, as (lig, pocket) pairs: () | (hist,) | (hist, hist2)."""
        return tuple(st[k] for k in ('hist', 'hist2') if k in st)

    def _joint_graph(self, st, kind, z_lig, z_pocket, first_s):
        g = st['graphs'].get(kind)
        if g is not None:
            return g
        device = z_lig.device
        run = self._joint_step(st, kind)

        def reset():
            self._joint_start(st, z_lig, z_pocket, first_s)

        rng = torch.cuda.get_rng_state(device)
        side = torch.cuda.Stream(device=device)
        side.wait_stream(torch.cuda.current_stream(device))
        reset()
        with torch.cuda.stream(side):
            run()                                   # warm-up: allocator, plan cache, workspace
        torch.cuda.current_stream(device).wait_stream(side)
        torch.cuda.set_rng_state(rng, device)
        reset()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            run()
        reset()
        sig = self.dynamics.capture_signature()
        if st['sig'] is not None and st['sig'] != sig:
            st['graphs'] = {}
        st['graphs'][kind] = g
        st['sig'] = sig
        return g

    def _graphed_joint_reverse_steps(self, z_lig, z_pocket, lig_mask, pocket_mask, n_samples, first_s, n_steps, timesteps):
        """Runs joint reverse steps s = first_s, first_s-1, ..., first_s-n_steps+1 by replaying one captured step (the
        joint counterpart of ConditionalDDPM._graphed_reverse_steps)."""
        dyn = self.dynamics
        st = self._joint_engine(z_lig, z_pocket, lig_mask, pocket_mask, n_samples, timesteps, 1)
        prev_defer, dyn.defer_status_check = dyn.defer_status_check, True
        try:
            g = self._joint_graph(st, 'reverse', z_lig, z_pocket, first_s)
            self._joint_start(st, z_lig, z_pocket, first_s)
            for _ in range(n_steps):
                g.replay()
        finally:
            dyn.defer_status_check = prev_defer
        dyn.check_status()
        return st['zl'].clone(), st['zp'].clone()

    def _graphed_joint_fast_loop(self, z_lig, z_pocket, lig_mask, pocket_mask, n_samples, timesteps, sampler, eta,
                                 return_frames, out_lig, out_pocket):
        """The whole 'ddim' / 'dpmpp_2m' / 'dpmpp_3m' reverse loop as ``timesteps`` replays of one captured step; frames are
        copied from the static state between replays, so the history of the multistep samplers runs through them."""
        dyn = self.dynamics
        st = self._joint_engine(z_lig, z_pocket, lig_mask, pocket_mask, n_samples, timesteps, 1, sampler, eta)
        s0 = timesteps - 1
        prev_defer, dyn.defer_status_check = dyn.defer_status_check, True
        try:
            g = self._joint_graph(st, sampler, z_lig, z_pocket, s0)
            self._joint_start(st, z_lig, z_pocket, s0)
            for s in reversed(range(timesteps)):
                g.replay()
                if (s * return_frames) % timesteps == 0:
                    idx = (s * return_frames) // timesteps
                    out_lig[idx], out_pocket[idx] = self.unnormalize_z(st['zl'], st['zp'])
        finally:
            dyn.defer_status_check = prev_defer
        dyn.check_status()
        return st['zl'].clone(), st['zp'].clone()

    def _joint_fast_step(self, s, t, row, zl, zp, hl, hp, lig_mask, pocket_mask, sampler, eta, u=0, commit=True):
        """Eager step z_t -> z_s of the joint model for any sampler (DESIGN §13, §15): 'ddpm' is sample_p_zs_given_zt at
        s = ``row`` (the s/T array) and t; for 'ddim' / 'dpmpp_2m' / 'dpmpp_3m' ``row`` [1, k] is the step's row of
        _fast_tables.  ``hl``, ``hp``: the history of each part (_empty_history).  Returns (z_lig, z_pocket, hist_lig,
        hist_pocket): with ``commit`` the history multistep_update writes, else the one given; either way moved by the step's
        joint COM removal, so that it stays in the frame of z.  ``u``: the RePaint block of the seeded reverse draw."""
        from . import seeded
        if sampler == 'ddpm':
            self._draw_at(seeded.STAGE_LOOP, s, u, seeded.PURPOSE_REVERSE)
            return (*self.sample_p_zs_given_zt(row, t, zl, zp, lig_mask, pocket_mask), hl, hp)
        nd = self.n_dims
        c = row.expand(t.shape[0], -1)
        cl, cp = c[lig_mask], c[pocket_mask]
        eps_l, eps_p = self.dynamics(zl, zp, t, lig_mask, pocket_mask)
        if sampler == 'ddim':
            mu_l = zl / cl[:, 0:1] - cl[:, 1:2] * eps_l
            mu_p = zp / cp[:, 0:1] - cp[:, 1:2] * eps_p
            if eta > 0:
                self._draw_at(seeded.STAGE_LOOP, s, u, seeded.PURPOSE_REVERSE)
                mu_l, mu_p = self.sample_normal(mu_l, mu_p, c[:, 2:3], lig_mask, pocket_mask)
            zl, zp = self._project_joint_com(mu_l, mu_p, lig_mask, pocket_mask)
            return zl, zp, hl, hp
        zl, new_l = multistep_update(zl, eps_l, hl, cl)
        zp, new_p = multistep_update(zp, eps_p, hp, cp)
        if commit:
            hl, hp = new_l, new_p
        else:
            hl, hp = tuple(x.clone() for x in hl), tuple(x.clone() for x in hp)
        mean = scatter_mean(torch.cat((zl[:, :nd], zp[:, :nd])), torch.cat((lig_mask, pocket_mask)), dim=0,
                            dim_size=t.shape[0])
        for x, m in ((zl, lig_mask), (zp, pocket_mask), *((x, lig_mask) for x in hl), *((x, pocket_mask) for x in hp)):
            x[:, :nd] -= mean[m]
        return zl, zp, hl, hp

    def _joint_fast_inpaint_step(self, s, i, t, row, gamma_s, z_lig, z_pocket, hist, xh0_lig, xh0_pocket, lig_fixed,
                                 pocket_fixed, lsel, psel, lmask, pmask, sampler, eta, commit):
        """Eager RePaint iteration (s, block i) of the joint inpaint (DESIGN §14), without the jump back (_joint_renoise): the
        known part, the reverse step (_joint_fast_step with ``t`` and ``row``), the COM alignment and the blend.  ``hist``:
        () for 'ddpm' and DDIM; for the multistep samplers (hist_lig, hist_pocket) as _joint_fast_step takes them, committed
        by the last iteration of step s + 1, in the frame of z.  The multistep COM removal moves it with z; the blend keeps the
        frame of the unknown part, so nothing else moves it; ``commit``: this iteration writes the history
        (multistep_update).  Returns (z_lig, z_pocket, hist)."""
        from . import seeded
        nd = self.n_dims
        # known nodes: forward-noised data; unknown nodes: one reverse step (en_diffusion.py:741-749)
        self._draw_at(seeded.STAGE_LOOP, s, i, seeded.PURPOSE_KNOWN)
        zk_lig, zk_pocket, _, _ = self.noised_representation(xh0_lig, xh0_pocket, lmask, pmask, gamma_s)
        zu_lig, zu_pocket, hl, hp = self._joint_fast_step(s, t, row, z_lig, z_pocket, *(hist or ((), ())), lmask, pmask, sampler,
                                                          eta, i, commit)
        hist = (hl, hp) if hl else ()
        # align the COM of the noised known part with the denoised one (en_diffusion.py:751-772)
        shift = self._fixed_com(zu_lig[:, :nd], zu_pocket[:, :nd], lsel, psel, lmask, pmask) - \
            self._fixed_com(zk_lig[:, :nd], zk_pocket[:, :nd], lsel, psel, lmask, pmask)
        zk_lig[:, :nd] = zk_lig[:, :nd] + shift[lmask]
        zk_pocket[:, :nd] = zk_pocket[:, :nd] + shift[pmask]
        z_lig = zk_lig * lig_fixed + zu_lig * (1 - lig_fixed)
        z_pocket = zk_pocket * pocket_fixed + zu_pocket * (1 - pocket_fixed)
        return z_lig, z_pocket, hist

    def _joint_renoise(self, z_lig, z_pocket, hist, gamma_t, gamma_s, lmask, pmask):
        """sample_p_zt_given_zs (the jump back, en_diffusion.py:790-807) with the multistep history ``hist`` (or ()) moved by
        the same joint COM removal: (hist_lig, hist_pocket), as _joint_fast_inpaint_step keeps it."""
        if not hist:
            return (*self.sample_p_zt_given_zs(z_lig, z_pocket, lmask, pmask, gamma_t, gamma_s), ())
        hl, hp = hist
        nd = self.n_dims
        _, sigma_ts, alpha_ts = self.sigma_and_alpha_t_given_s(gamma_t, gamma_s, z_lig)
        zl, zp = self.sample_normal(alpha_ts[lmask] * z_lig, alpha_ts[pmask] * z_pocket, sigma_ts, lmask, pmask)
        mean = scatter_mean(torch.cat((zl[:, :nd], zp[:, :nd])), torch.cat((lmask, pmask)), dim=0)

        def move(x, m):
            x = x.clone()
            x[:, :nd] = x[:, :nd] - mean[m]
            return x
        return (move(zl, lmask), move(zp, pmask), (tuple(move(x, lmask) for x in hl), tuple(move(x, pmask) for x in hp)))

    @follows_dynamics_determinism
    @torch.no_grad()
    def sample(self, n_samples, num_nodes_lig, num_nodes_pocket, return_frames=1, timesteps=None, device='cpu', seeds=None,
               sampler='ddpm', eta=0.0):
        """en_diffusion.py:581-651: unconditional joint sampling of ligand and pocket.  ``seeds``: one int64 per sample
        (seeded.py); every draw then comes from the sample's own seed instead of torch's global generator.  ``sampler``:
        'ddpm' (the reference's ancestral step), 'ddim' (with noise level ``eta`` in [0, 1]), 'dpmpp_2m' or 'dpmpp_3m', on
        the same ``timesteps`` grid (DESIGN §13, §15)."""
        from . import seeded
        check_sampler(sampler, eta)
        seeds = seeded.as_seeds(seeds, n_samples, device)
        lig_mask = num_nodes_to_batch_mask(n_samples, num_nodes_lig, device)
        pocket_mask = num_nodes_to_batch_mask(n_samples, num_nodes_pocket, device)
        with self._seeded(seeds, lig_mask, pocket_mask):
            return self._sample(n_samples, lig_mask, pocket_mask, return_frames, timesteps, sampler, float(eta))

    def _sample(self, n_samples, lig_mask, pocket_mask, return_frames, timesteps, sampler='ddpm', eta=0.0):
        from . import seeded
        timesteps = self.T if timesteps is None else timesteps
        assert 0 < return_frames <= timesteps and timesteps % return_frames == 0
        if self._rng is not None:
            seeded.check_schedule(timesteps)
        combined_mask = torch.cat((lig_mask, pocket_mask))
        self._draw_at(seeded.STAGE_PRIOR)
        z_lig, z_pocket = self.sample_combined_position_feature_noise(lig_mask, pocket_mask)
        self.assert_mean_zero_with_mask(torch.cat((z_lig[:, :self.n_dims], z_pocket[:, :self.n_dims])), combined_mask)
        out_lig = torch.zeros((return_frames,) + z_lig.size(), device=z_lig.device)
        out_pocket = torch.zeros((return_frames,) + z_pocket.size(), device=z_pocket.device)
        use_graph = self._joint_use_graph(z_lig.device)
        if use_graph and sampler != 'ddpm':
            z_lig, z_pocket = self._graphed_joint_fast_loop(z_lig, z_pocket, lig_mask, pocket_mask, n_samples, timesteps, sampler,
                                                            eta, return_frames, out_lig, out_pocket)
        elif use_graph:
            stride = timesteps // return_frames       # frames are saved at s = idx * stride
            s_hi = timesteps - 1
            while s_hi >= 0:
                s_lo = (s_hi // stride) * stride
                z_lig, z_pocket = self._graphed_joint_reverse_steps(
                    z_lig, z_pocket, lig_mask, pocket_mask, n_samples, s_hi, s_hi - s_lo + 1, timesteps)
                out_lig[s_lo // stride], out_pocket[s_lo // stride] = self.unnormalize_z(z_lig, z_pocket)
                s_hi = s_lo - 1
        else:
            fast = None if sampler == 'ddpm' else self._fast_tables(timesteps, sampler, eta, z_lig.device)
            h_lig, h_pocket = self._empty_history(z_lig, sampler), self._empty_history(z_pocket, sampler)
            for s in reversed(range(0, timesteps)):
                t, row = self._eager_row(s, timesteps, n_samples, z_lig.device, fast)
                z_lig, z_pocket, h_lig, h_pocket = self._joint_fast_step(s, t, row, z_lig, z_pocket, h_lig, h_pocket, lig_mask,
                                                                         pocket_mask, sampler, eta)
                if (s * return_frames) % timesteps == 0:
                    idx = (s * return_frames) // timesteps
                    out_lig[idx], out_pocket[idx] = self.unnormalize_z(z_lig, z_pocket)
        self.assert_mean_zero_with_mask(torch.cat((z_lig[:, :self.n_dims], z_pocket[:, :self.n_dims])), combined_mask)
        self._draw_at(seeded.STAGE_FINAL)
        x_lig, h_lig, x_pocket, h_pocket = self.sample_p_xh_given_z0(z_lig, z_pocket, lig_mask, pocket_mask, n_samples)
        self.assert_mean_zero_with_mask(torch.cat((x_lig, x_pocket), dim=0), combined_mask)
        if return_frames == 1:
            x_lig, x_pocket = self._project_joint_cog_drift(x_lig, x_pocket, lig_mask, pocket_mask)
        out_lig[0] = torch.cat([x_lig, h_lig], dim=1)
        out_pocket[0] = torch.cat([x_pocket, h_pocket], dim=1)
        return out_lig.squeeze(0), out_pocket.squeeze(0), lig_mask, pocket_mask

    @staticmethod
    def _empty_history(x, sampler):
        """The zero history of one part for the eager steps, x0_hat tensors newest first: (m1,) for 'dpmpp_2m', (m1, m2) for
        'dpmpp_3m', () for the samplers without one."""
        return (torch.zeros_like(x),) * {'dpmpp_2m': 1, 'dpmpp_3m': 2}.get(sampler, 0)

    # ---- RePaint-style inpainting with the joint model (en_diffusion.py:653-837) ---------------------------------
    @staticmethod
    def get_repaint_schedule(resamplings, jump_length, timesteps):
        """en_diffusion.py:653-674: number of consecutive denoising steps before each jump back, in execution order."""
        blocks = []
        done = 0
        while done < timesteps:
            step = jump_length if done + jump_length < timesteps else timesteps - done
            if blocks:
                blocks[-1] += step
                if step == jump_length and done + jump_length < timesteps:
                    blocks.extend([jump_length] * (resamplings - 1))
            else:
                blocks.extend([jump_length] * resamplings if done + jump_length < timesteps else [step])
            done += step
        return blocks[::-1]

    def _project_joint_cog_drift(self, x_lig, x_pocket, lig_mask, pocket_mask):
        combined_mask = torch.cat((lig_mask, pocket_mask))
        xc = torch.cat((x_lig, x_pocket))

        def project():
            xp = self.remove_mean_batch(xc, combined_mask)
            return xp[:len(x_lig)], xp[len(x_lig):]
        return self._project_cog_drift(x_lig, x_pocket, lig_mask, project, pocket_mask, xc, combined_mask)

    def _fixed_com(self, x_lig, x_pocket, lig_sel, pocket_sel, lig_mask, pocket_mask):
        """COM of the fixed ligand+pocket nodes per graph."""
        return scatter_mean(torch.cat((x_lig[lig_sel], x_pocket[pocket_sel])),
                            torch.cat((lig_mask[lig_sel], pocket_mask[pocket_sel])), dim=0)

    @follows_dynamics_determinism
    @torch.no_grad()
    def inpaint(self, ligand, pocket, lig_fixed, pocket_fixed, resamplings=1, jump_length=1, return_frames=1,
                timesteps=None, seeds=None, sampler='ddpm', eta=0.0):
        """en_diffusion.py:677-837: sample the free nodes while the fixed ones follow q(z_s | x).  ``seeds``: as sample.
        ``sampler`` / ``eta``: the reverse step of every RePaint iteration, as sample; 'dpmpp_2m' and 'dpmpp_3m' need
        jump_length = 1 (DESIGN §14, §15).  With every pocket node fixed this is how a joint model generates a ligand for a given pocket in few
        steps."""
        from . import seeded
        check_sampler(sampler, eta)
        if sampler in MULTISTEP and jump_length > 1:
            raise ValueError(f"sampler={sampler!r} needs jump_length = 1 (got {jump_length}): its history has no rule for "
                             f"jumps over several steps; use 'ddim'")
        seeds = seeded.as_seeds(seeds, len(ligand['size']), ligand['x'].device)
        with self._seeded(seeds, ligand['mask'], pocket['mask']):
            return self._inpaint(ligand, pocket, lig_fixed, pocket_fixed, resamplings, jump_length, return_frames, timesteps,
                                 sampler, float(eta))

    def _inpaint(self, ligand, pocket, lig_fixed, pocket_fixed, resamplings, jump_length, return_frames, timesteps,
                 sampler='ddpm', eta=0.0):
        from . import seeded
        timesteps = self.T if timesteps is None else timesteps
        if self._rng is not None:          # u counts the jump-back blocks of the RePaint schedule
            seeded.check_schedule(timesteps, len(self.get_repaint_schedule(resamplings, jump_length, timesteps)))
        assert 0 < return_frames <= timesteps
        assert timesteps % return_frames == 0
        assert jump_length == 1 or return_frames == 1, "Chain visualization is only implemented for jump_length=1"
        if len(lig_fixed.size()) == 1:
            lig_fixed = lig_fixed.unsqueeze(1)
        if len(pocket_fixed.size()) == 1:
            pocket_fixed = pocket_fixed.unsqueeze(1)
        ligand, pocket = self.normalize(ligand, pocket)
        lmask, pmask = ligand['mask'], pocket['mask']
        lsel, psel = lig_fixed.bool().view(-1), pocket_fixed.bool().view(-1)
        n_samples = len(ligand['size'])
        nd = self.n_dims
        combined_mask = torch.cat((lmask, pmask))
        xh0_lig = torch.cat([ligand['x'], ligand['one_hot']], dim=1)
        xh0_pocket = torch.cat([pocket['x'], pocket['one_hot']], dim=1)

        # centre the system on the COM of the known nodes (en_diffusion.py:707-717)
        mean_known = self._fixed_com(ligand['x'], pocket['x'], lsel, psel, lmask, pmask)
        xh0_lig[:, :nd] = xh0_lig[:, :nd] - mean_known[lmask]
        xh0_pocket[:, :nd] = xh0_pocket[:, :nd] - mean_known[pmask]

        self._draw_at(seeded.STAGE_PRIOR)
        z_lig, z_pocket = self.sample_combined_position_feature_noise(lmask, pmask)
        out_lig = torch.zeros((return_frames,) + z_lig.size(), device=z_lig.device)
        out_pocket = torch.zeros((return_frames,) + z_pocket.size(), device=z_pocket.device)

        schedule = self.get_repaint_schedule(resamplings, jump_length, timesteps)
        s = timesteps - 1
        if self._joint_use_graph(z_lig.device):
            dyn = self.dynamics
            st = self._joint_engine(z_lig, z_pocket, lmask, pmask, n_samples, timesteps, jump_length, sampler, eta)
            multistep = sampler in MULTISTEP
            if st['known'] is None:       # static buffers the captured RePaint iteration reads
                st['known'] = dict(xl=torch.empty_like(xh0_lig), xp=torch.empty_like(xh0_pocket),
                                   fl=torch.empty(len(lmask), device=z_lig.device), fp=torch.empty(len(pmask), device=z_lig.device))
            kn = st['known']
            kn['xl'].copy_(xh0_lig); kn['xp'].copy_(xh0_pocket); kn['fl'].copy_(lig_fixed.view(-1)); kn['fp'].copy_(pocket_fixed.view(-1))
            prev_defer, dyn.defer_status_check = dyn.defer_status_check, True
            try:
                g_it = self._joint_graph(st, 'inpaint', z_lig, z_pocket, s)
                g_jump = self._joint_graph(st, 'inpaint_jump', z_lig, z_pocket, s) if len(schedule) > 1 else None
                # 2M / 3M: the frame-before-jump path replays an iteration that does not commit (captured here: a capture
                # resets the static state)
                g_hold = self._joint_graph(st, 'inpaint_hold', z_lig, z_pocket, s) if multistep and len(schedule) > 1 else None
                self._joint_start(st, z_lig, z_pocket, s)
                for i, n_denoise in enumerate(schedule):
                    for j in range(n_denoise):
                        jump = j == n_denoise - 1 and i < len(schedule) - 1
                        frame = (n_denoise > jump_length or i == len(schedule) - 1) and (s * return_frames) % timesteps == 0
                        # a frame is taken after the blend and BEFORE the jump back (en_diffusion.py:777-788): in that case the
                        # jump runs as eager torch ops on the static state instead of inside the fused kernel (2M / 3M: after
                        # an iteration that does not commit)
                        if jump and frame and multistep:
                            g_hold.replay()
                        else:
                            (g_jump if (jump and not frame) else g_it).replay()
                        if frame:
                            idx = (s * return_frames) // timesteps
                            out_lig[idx], out_pocket[idx] = self.unnormalize_z(st['zl'], st['zp'])
                        if jump:
                            if frame:
                                self._draw_at(seeded.STAGE_LOOP, s, i, seeded.PURPOSE_RENOISE)
                                s_arr = torch.full((n_samples, 1), fill_value=s, device=z_lig.device) / timesteps
                                t_back = torch.full((n_samples, 1), fill_value=s + jump_length, device=z_lig.device) / timesteps
                                g_t = self.inflate_batch_array(self.gamma(t_back), ligand['x'])
                                g_s = self.inflate_batch_array(self.gamma(s_arr), ligand['x'])
                                hists = self._joint_static_history(st)
                                hist = (tuple(h[0] for h in hists), tuple(h[1] for h in hists)) if hists else ()
                                zl, zp, moved = self._joint_renoise(st['zl'], st['zp'], hist, g_t, g_s, lmask, pmask)
                                for x, y in zip(sum(hist, ()), sum(moved, ())):
                                    x.copy_(y)
                                st['zl'].copy_(zl); st['zp'].copy_(zp); st['step'].add_(jump_length)
                                if st['seeded']:
                                    st['u'].add_(1)
                            s = s + jump_length
                        s -= 1
            finally:
                dyn.defer_status_check = prev_defer
            dyn.check_status()
            z_lig, z_pocket = st['zl'].clone(), st['zp'].clone()
            self.assert_mean_zero_with_mask(torch.cat((z_lig[:, :nd], z_pocket[:, :nd]), dim=0), combined_mask)
        else:
            if sampler != 'ddpm':
                t_table, coef = self._fast_tables(timesteps, sampler, eta, z_lig.device)
            hist = ()
            if sampler in MULTISTEP:
                hist = (self._empty_history(z_lig, sampler), self._empty_history(z_pocket, sampler))
            for i, n_denoise in enumerate(schedule):
                for j in range(n_denoise):
                    jump = j == n_denoise - 1 and i < len(schedule) - 1
                    s_array = torch.full((n_samples, 1), fill_value=s, device=z_lig.device)
                    t_array = (s_array + 1) / timesteps
                    s_array = s_array / timesteps
                    gamma_s = self.inflate_batch_array(self.gamma(s_array), ligand['x'])
                    t, row = (t_array, s_array) if sampler == 'ddpm' else (t_table[s].expand(n_samples, 1), coef[s:s + 1])
                    z_lig, z_pocket, hist = self._joint_fast_inpaint_step(
                        s, i, t, row, gamma_s, z_lig, z_pocket, hist, xh0_lig, xh0_pocket, lig_fixed, pocket_fixed, lsel, psel,
                        lmask, pmask, sampler, eta, not jump)
                    self.assert_mean_zero_with_mask(torch.cat((z_lig[:, :nd], z_pocket[:, :nd]), dim=0), combined_mask)
                    if (n_denoise > jump_length or i == len(schedule) - 1) and (s * return_frames) % timesteps == 0:
                        idx = (s * return_frames) // timesteps
                        out_lig[idx], out_pocket[idx] = self.unnormalize_z(z_lig, z_pocket)
                    if jump:                                           # jump back jump_length steps
                        t_back = torch.full((n_samples, 1), fill_value=s + jump_length, device=z_lig.device) / timesteps
                        gamma_t = self.inflate_batch_array(self.gamma(t_back), ligand['x'])
                        self._draw_at(seeded.STAGE_LOOP, s, i, seeded.PURPOSE_RENOISE)
                        z_lig, z_pocket, hist = self._joint_renoise(z_lig, z_pocket, hist, gamma_t, gamma_s, lmask, pmask)
                        s = s + jump_length
                    s -= 1

        self._draw_at(seeded.STAGE_FINAL)
        x_lig, h_lig, x_pocket, h_pocket = self.sample_p_xh_given_z0(z_lig, z_pocket, lmask, pmask, n_samples)
        self.assert_mean_zero_with_mask(torch.cat((x_lig, x_pocket), dim=0), combined_mask)
        if return_frames == 1:
            x_lig, x_pocket = self._project_joint_cog_drift(x_lig, x_pocket, lmask, pmask)
        out_lig[0] = torch.cat([x_lig, h_lig], dim=1)
        out_pocket[0] = torch.cat([x_pocket, h_pocket], dim=1)
        return out_lig.squeeze(0), out_pocket.squeeze(0), lmask, pmask

    # ---- evaluation-mode variational bound (en_diffusion.py:109-261, :319-469) ---------------------------------------
    @staticmethod
    def gaussian_KL(q_mu_minus_p_mu_squared, q_sigma, p_sigma, d):
        """KL(N(mu_q, q_sigma^2 I_d) || N(mu_p, p_sigma^2 I_d)) from ||mu_q - mu_p||^2 (en_diffusion.py:840-853)."""
        log_ratio = torch.log(p_sigma / q_sigma)
        return d * log_ratio + 0.5 * (d * q_sigma ** 2 + q_mu_minus_p_mu_squared) / (p_sigma ** 2) - 0.5 * d

    @staticmethod
    def cdf_standard_gaussian(x):
        return 0.5 * (1. + torch.erf(x / math.sqrt(2)))

    def log_pN(self, N_lig, N_pocket):
        """log p(N) of the joint size prior, so that -log p(x, h, N) = -log p(x, h | N) - log p(N)."""
        return self.size_distribution.log_prob(N_lig, N_pocket)

    def delta_log_px(self, num_nodes):
        """Log-volume change of the coordinate normalisation x / norm_values[0] on the x subspace."""
        return -self.subspace_dimensionality(num_nodes) * np.log(self.norm_values[0])

    def log_constants_p_x_given_z0(self, n_nodes, device):
        """The sigma_0-dependent constants of log p(x | z_0): sigma_x = SNR(-gamma_0 / 2) per dimension."""
        n = len(n_nodes)
        dof = self.subspace_dimensionality(n_nodes)
        log_sigma_x = 0.5 * self.gamma(torch.zeros((n, 1), device=device)).view(n)
        return dof * (-log_sigma_x - 0.5 * np.log(2 * np.pi))

    def _kl_prior_from_norms(self, mu_norm2_x, mu_norm2_h, num_nodes, device):
        """KL(q(z_T | x, h) || N(0, I)) from ||alpha_T x||^2 and ||alpha_T h||^2 per graph."""
        gamma_T = self.gamma(torch.ones((len(num_nodes), 1), device=device))
        sigma_T = self.sigma(gamma_T, gamma_T).view(-1)
        ones = torch.ones_like(sigma_T)
        kl_h = self.gaussian_KL(mu_norm2_h, sigma_T, ones, d=1)
        kl_x = self.gaussian_KL(mu_norm2_x, sigma_T, ones, self.subspace_dimensionality(num_nodes))
        return kl_x + kl_h

    def kl_prior_with_pocket(self, xh_lig, xh_pocket, mask_lig, mask_pocket, num_nodes):
        """en_diffusion.py:109-155: KL of q(z_T | x, h) of ligand and pocket against the standard normal prior."""
        nd = self.n_dims
        alpha_T = self.alpha(self.gamma(torch.ones((len(num_nodes), 1), device=xh_lig.device)), xh_lig)
        mu_lig, mu_pocket = alpha_T[mask_lig] * xh_lig, alpha_T[mask_pocket] * xh_pocket
        norm_x = self.sum_except_batch(mu_lig[:, :nd] ** 2, mask_lig) + self.sum_except_batch(mu_pocket[:, :nd] ** 2, mask_pocket)
        norm_h = self.sum_except_batch(mu_lig[:, nd:] ** 2, mask_lig) + self.sum_except_batch(mu_pocket[:, nd:] ** 2, mask_pocket)
        return self._kl_prior_from_norms(norm_x, norm_h, num_nodes, xh_lig.device)

    def _log_ph_given_z0(self, one_hot, z_h, sigma_0_cat, mask, epsilon=1e-10):
        """Discretised-Gaussian likelihood of the one-hot types given z_0.h, summed per graph (en_diffusion.py:216-255)."""
        target = one_hot * self.norm_values[1] + self.norm_biases[1]
        centred = (z_h * self.norm_values[1] + self.norm_biases[1]) - 1
        width = sigma_0_cat[mask]
        log_p = torch.log(self.cdf_standard_gaussian((centred + 0.5) / width)
                          - self.cdf_standard_gaussian((centred - 0.5) / width) + epsilon)
        log_p = log_p - torch.logsumexp(log_p, dim=1, keepdim=True)
        return self.sum_except_batch(log_p * target, mask)

    def log_pxh_given_z0_without_constants(self, ligand, z_0_lig, eps_lig, net_out_lig, pocket, z_0_pocket, eps_pocket,
                                           net_out_pocket, gamma_0, epsilon=1e-10):
        """en_diffusion.py:185-261: -1/2 |eps_0.x - net_0.x|^2 of ligand and pocket, and log p(h | z_0) of both."""
        nd = self.n_dims
        sigma_0_cat = self.sigma(gamma_0, target_tensor=z_0_lig) * self.norm_values[1]
        log_px_lig = -0.5 * self.sum_except_batch((eps_lig[:, :nd] - net_out_lig[:, :nd]) ** 2, ligand['mask'])
        log_px_pocket = -0.5 * self.sum_except_batch((eps_pocket[:, :nd] - net_out_pocket[:, :nd]) ** 2, pocket['mask'])
        log_ph = self._log_ph_given_z0(ligand['one_hot'], z_0_lig[:, nd:], sigma_0_cat, ligand['mask'], epsilon) + \
            self._log_ph_given_z0(pocket['one_hot'], z_0_pocket[:, nd:], sigma_0_cat, pocket['mask'], epsilon)
        return log_px_lig, log_px_pocket, log_ph

    @staticmethod
    def _eps_hat_mean(net_out, mask, n_graphs):
        """Mean over graphs of the per-graph mean |net_out| (the ``info`` entries of forward)."""
        return scatter_mean(net_out.abs().mean(1), mask, dim=0, dim_size=n_graphs).mean()

    def _vlb_native(self, device) -> bool:
        """Evaluation-mode forward on the native kernels: 'auto' on CUDA with the native EGNNDynamics; 'eager' keeps the
        reference-order torch ops; 'graph' insists on the native path."""
        from .dynamics import EGNNDynamics
        if self.loop_engine == 'eager':
            return False
        ok = isinstance(self.dynamics, EGNNDynamics) and torch.device(device).type == 'cuda'
        if self.loop_engine == 'graph' and not ok:
            raise RuntimeError("loop_engine='graph' needs the native EGNNDynamics on a CUDA device")
        return ok

    def _native_denoise_pair(self, z_t, t, z_0, t_0, lig_mask, pocket_mask):
        """The two denoiser calls of the eval forward (at t and at 0) with one NaN check after both."""
        dyn = self.dynamics
        prev, dyn.defer_status_check = dyn.defer_status_check, True
        try:
            net_t = dyn(z_t[0], z_t[1], t, lig_mask, pocket_mask)
            net_0 = dyn(z_0[0], z_0[1], t_0, lig_mask, pocket_mask)
        finally:
            dyn.defer_status_check = prev
        dyn.check_status()
        return net_t, net_0

    def _native_noise(self, xh_lig, eps_lig, xh_pocket, eps_pocket, lig_mask, pocket_mask, gamma):
        """z = alpha xh + sigma eps per graph in one launch (libdiffsbdd_b200 dsb_ddpm_noise); pocket skipped if None."""
        from . import _native
        lib = _native.load()
        coef = torch.cat([self.alpha(gamma, gamma), self.sigma(gamma, gamma)], dim=1).float().contiguous()
        z_lig = torch.empty_like(xh_lig)
        z_pocket = None if xh_pocket is None else torch.empty_like(xh_pocket)
        ptr = lambda x: None if x is None else x.data_ptr()
        _native.check(lib.dsb_ddpm_noise(
            ptr(xh_lig), ptr(eps_lig), ptr(xh_pocket), ptr(eps_pocket), ptr(coef), ptr(lig_mask), ptr(pocket_mask),
            len(lig_mask), len(pocket_mask), coef.shape[0], self.atom_nf, self.residue_nf, ptr(z_lig), ptr(z_pocket),
            torch.cuda.current_stream(xh_lig.device).cuda_stream))
        return z_lig, z_pocket

    def _native_vlb_terms(self, lig, pocket, lig_mask, pocket_mask, gamma_t, gamma_0, vnode_idx):
        """One dsb_ddpm_vlb_terms launch.  lig = (xh0, z_t, eps_t, net_t, z_0, eps_0, net_0); pocket = (xh0, eps_t, net_t, z_0,
        eps_0, net_0) or None (ligand-only likelihood).  Returns the per-graph sums [n_graphs, 11] and xh_lig_hat."""
        from . import _native
        lib = _native.load()
        n = gamma_t.shape[0]
        device = lig[0].device
        gamma_T = self.gamma(torch.ones((n, 1), device=device))
        coef = torch.cat([self.alpha(gamma_T, gamma_T), self.sigma(gamma_0, gamma_0) * self.norm_values[1],
                          self.alpha(gamma_t, gamma_t), self.sigma(gamma_t, gamma_t)], dim=1).float().contiguous()
        lig = [x.float().contiguous() for x in lig]
        pocket = [None] * 6 if pocket is None else [x.float().contiguous() for x in pocket]
        terms = torch.empty((n, 11), device=device)
        xh_lig_hat = torch.empty_like(lig[1])
        ptr = lambda x: None if x is None else x.data_ptr()
        _native.check(lib.dsb_ddpm_vlb_terms(
            *[ptr(x) for x in lig], *[ptr(x) for x in pocket], ptr(coef), ptr(lig_mask), ptr(pocket_mask), len(lig_mask),
            len(pocket_mask), n, self.atom_nf, self.residue_nf, float(self.norm_values[1]), float(self.norm_biases[1]),
            -1 if vnode_idx is None else int(vnode_idx), ptr(terms), ptr(xh_lig_hat),
            torch.cuda.current_stream(device).cuda_stream))
        return terms, xh_lig_hat

    @follows_dynamics_determinism
    @torch.no_grad()
    def forward(self, ligand, pocket, return_info=False):
        """Eval-mode variational bound of the joint model (en_diffusion.py:336-469): the terms of -log p(x, h | N) for
        ligand and pocket at one random t in [1, T] plus the t = 0 reconstruction term.  RNG calls as the reference:
        randint for t, then the noise at t, then the noise at 0.  Training (t = 0 sampling, autograd) is not built."""
        if self.training:
            raise NotImplementedError('the training loss is not built (no backward kernels); call eval() for the NLL bound')
        ligand, pocket = self.normalize(ligand, pocket)
        lm, pm = ligand['mask'], pocket['mask']
        n, device, nd = ligand['size'].size(0), ligand['x'].device, self.n_dims
        n_nodes = ligand['size'] + pocket['size']
        delta_log_px = self.delta_log_px(n_nodes)
        t_int = torch.randint(1, self.T + 1, size=(n, 1), device=device).float()
        s, t = (t_int - 1) / self.T, t_int / self.T
        t_0 = torch.zeros_like(s)
        gamma_s = self.inflate_batch_array(self.gamma(s), ligand['x'])
        gamma_t = self.inflate_batch_array(self.gamma(t), ligand['x'])
        gamma_0 = self.inflate_batch_array(self.gamma(t_0), ligand['x'])
        xh_lig = torch.cat([ligand['x'], ligand['one_hot']], dim=1)
        xh_pocket = torch.cat([pocket['x'], pocket['one_hot']], dim=1)
        SNR_weight = (1 - self.SNR(gamma_s - gamma_t)).squeeze(1)
        neg_log_constants = -self.log_constants_p_x_given_z0(n_nodes=n_nodes, device=device)

        if self._vlb_native(device):
            eps_t = self.sample_combined_position_feature_noise(lm, pm)
            z_t = self._native_noise(xh_lig, eps_t[0], xh_pocket, eps_t[1], lm, pm, gamma_t)
            eps_0 = self.sample_combined_position_feature_noise(lm, pm)
            z_0 = self._native_noise(xh_lig, eps_0[0], xh_pocket, eps_0[1], lm, pm, gamma_0)
            (net_t_lig, net_t_pocket), (net_0_lig, net_0_pocket) = self._native_denoise_pair(z_t, t, z_0, t_0, lm, pm)
            terms, xh_lig_hat = self._native_vlb_terms(
                (xh_lig, z_t[0], eps_t[0], net_t_lig, z_0[0], eps_0[0], net_0_lig),
                (xh_pocket, eps_t[1], net_t_pocket, z_0[1], eps_0[1], net_0_pocket), lm, pm, gamma_t, gamma_0, None)
            error_t_lig, error_t_pocket = terms[:, 0], terms[:, 1]
            loss_0_x_ligand, loss_0_x_pocket, loss_0_h = 0.5 * terms[:, 2], 0.5 * terms[:, 3], -terms[:, 4]
            kl_prior = self._kl_prior_from_norms(terms[:, 5], terms[:, 6], n_nodes, device)
            cnt_l = ligand['size'].clamp(min=1).float()
            cnt_p = pocket['size'].clamp(min=1).float()
            info = {'eps_hat_lig_x': (terms[:, 7] / (nd * cnt_l)).mean(),
                    'eps_hat_lig_h': (terms[:, 8] / (self.atom_nf * cnt_l)).mean(),
                    'eps_hat_pocket_x': (terms[:, 9] / (nd * cnt_p)).mean(),
                    'eps_hat_pocket_h': (terms[:, 10] / (self.residue_nf * cnt_p)).mean()}
        else:
            z_t_lig, z_t_pocket, eps_t_lig, eps_t_pocket = self.noised_representation(xh_lig, xh_pocket, lm, pm, gamma_t)
            net_t_lig, net_t_pocket = self.dynamics(z_t_lig, z_t_pocket, t, lm, pm)
            xh_lig_hat = self.xh_given_zt_and_epsilon(z_t_lig, net_t_lig, gamma_t, lm)
            error_t_lig = self.sum_except_batch((eps_t_lig - net_t_lig) ** 2, lm)
            error_t_pocket = self.sum_except_batch((eps_t_pocket - net_t_pocket) ** 2, pm)
            kl_prior = self.kl_prior_with_pocket(xh_lig, xh_pocket, lm, pm, n_nodes)
            z_0_lig, z_0_pocket, eps_0_lig, eps_0_pocket = self.noised_representation(xh_lig, xh_pocket, lm, pm, gamma_0)
            net_0_lig, net_0_pocket = self.dynamics(z_0_lig, z_0_pocket, t_0, lm, pm)
            log_px_lig, log_px_pocket, log_ph = self.log_pxh_given_z0_without_constants(
                ligand, z_0_lig, eps_0_lig, net_0_lig, pocket, z_0_pocket, eps_0_pocket, net_0_pocket, gamma_0)
            loss_0_x_ligand, loss_0_x_pocket, loss_0_h = -log_px_lig, -log_px_pocket, -log_ph
            info = {'eps_hat_lig_x': self._eps_hat_mean(net_t_lig[:, :nd], lm, n),
                    'eps_hat_lig_h': self._eps_hat_mean(net_t_lig[:, nd:], lm, n),
                    'eps_hat_pocket_x': self._eps_hat_mean(net_t_pocket[:, :nd], pm, n),
                    'eps_hat_pocket_h': self._eps_hat_mean(net_t_pocket[:, nd:], pm, n)}

        log_pN = self.log_pN(ligand['size'], pocket['size'])
        terms = (delta_log_px, error_t_lig, error_t_pocket, SNR_weight, loss_0_x_ligand, loss_0_x_pocket, loss_0_h,
                 neg_log_constants, kl_prior, log_pN, t_int.squeeze(), xh_lig_hat)
        return (*terms, info) if return_info else terms
