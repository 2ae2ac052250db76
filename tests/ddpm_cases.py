"""Shared definitions of the DDPM-wrapper parity cases (used by the golden generator and the tests)."""
import math

import torch

from diffsbdd_b200.config import DynamicsConfig
from diffsbdd_b200 import synthetic as syn
from oracle.cpu_denoiser import OracleDynamics  # noqa: F401

# small conditional denoiser (kernel-supported dims: H=64) so CPU loops stay fast
DDPM_CFG = DynamicsConfig(joint_nf=16, hidden_nf=64, n_layers=2)
HIST = [[0.0, 1.0, 2.0], [1.0, 3.0, 1.0], [2.0, 1.0, 0.5]]
N_POCKET = [22, 17]

SAMPLER_CASES = {
    'sample_T6': dict(kind='sample', T=6, timesteps=None, frames=1, n_lig=[7, 5], seed=101),
    'sample_T12_frames3_sub6': dict(kind='sample', T=12, timesteps=6, frames=3, n_lig=[4, 9], seed=102),
    'inpaint_T4_r2_ligand': dict(kind='inpaint', T=8, timesteps=4, resamplings=2, n_lig=[8, 6], n_fixed=3,
                                 center='ligand', seed=103),
    'inpaint_T3_r1_pocket': dict(kind='inpaint', T=3, timesteps=None, resamplings=1, n_lig=[5, 7], n_fixed=2,
                                 center='pocket', seed=104),
    'diversify_3of10': dict(kind='diversify', T=10, noising_steps=3, n_lig=[6, 6], seed=105),
}


# joint model (update_pocket_coords=True): EnVariationalDiffusion.sample / .inpaint (en_diffusion.py:839, :677)
JOINT_CFG = DynamicsConfig(joint_nf=16, hidden_nf=64, n_layers=2, update_pocket_coords=True)
JOINT_CASES = {
    'joint_sample_T5': dict(kind='sample', T=5, timesteps=None, frames=1, n_lig=[6, 4], seed=201),
    'joint_inpaint_T6_r2_j2': dict(kind='inpaint', T=6, timesteps=None, resamplings=2, jump_length=2, frames=1,
                                   n_lig=[7, 5], n_fixed=2, pocket_fixed=True, seed=202),
    'joint_inpaint_T8_sub4_frames2': dict(kind='inpaint', T=8, timesteps=4, resamplings=1, jump_length=1, frames=2,
                                          n_lig=[5, 6], n_fixed=0, pocket_fixed=True, seed=203),
    'joint_inpaint_T4_r3_partial_pocket': dict(kind='inpaint', T=4, timesteps=None, resamplings=3, jump_length=1,
                                               frames=1, n_lig=[6, 6], n_fixed=3, pocket_fixed=False, seed=204),
}


def make_pocket_fixed(spec, pocket):
    """0/1 per pocket node: all fixed, or every third node free (exercises the pocket blend of en_diffusion.py:775)."""
    f = torch.ones(len(pocket['mask']))
    if not spec['pocket_fixed']:
        f[::3] = 0
    return f


def make_pocket(device='cpu'):
    p = syn.synthetic_pocket(DDPM_CFG, N_POCKET, seed=31, spread=3.0)
    return {k: v.to(device) for k, v in p.items()}


def make_ligand(n_lig, n_fixed, device='cpu'):
    """Reference ``ligand`` dict + 0/1 ``lig_fixed`` (inpaint.py:117-141: first n_fixed atoms of every sample)."""
    g = torch.Generator().manual_seed(77)
    n = sum(n_lig)
    mask = torch.repeat_interleave(torch.arange(len(n_lig)), torch.tensor(n_lig))
    x = torch.randn((n, 3), generator=g) * 1.5
    types = torch.randint(0, DDPM_CFG.atom_nf, (n,), generator=g)
    fixed = torch.zeros(n)
    start = 0
    for k in n_lig:
        fixed[start:start + n_fixed] = 1
        start += k
    lig = {'x': x.to(device), 'one_hot': torch.nn.functional.one_hot(types, DDPM_CFG.atom_nf).float().to(device),
           'size': torch.tensor(n_lig, device=device), 'mask': mask.to(device)}
    return lig, fixed.to(device)


# per-graph (ligand rows, pocket rows) of the fused-kernel tests: each test's own small ragged batch, the configs[2] batch, and
# a batch with more than 128 ligand rows and 300 pocket rows in one graph (one 128-thread block per graph: strided row loops)
# next to a one-atom ligand
DDPM_SHAPES = {
    'ragged': None,
    'configs2': ([25] * 64, [175] * 64),
    'large': ([150, 1, 20], [300, 40, 9]),
}


def ddpm_shape(shape, ragged_lig, ragged_poc):
    return (ragged_lig, ragged_poc) if DDPM_SHAPES[shape] is None else DDPM_SHAPES[shape]


def assert_fp64_bound(got, want32, want64, what):
    """The kernel's max-abs error against the float64 evaluation of the same ops on the same fp32 inputs is at most twice the
    error of the fp32 torch ops, or 4 ulp of the output's largest magnitude, whichever is larger."""
    got, want32, want64 = (x.detach().cpu().double() for x in (got, want32, want64))
    err = float((got - want64).abs().max())
    err32 = float((want32 - want64).abs().max())
    big = float(want64.abs().max())
    ulp = 2.0 ** (math.floor(math.log2(big)) - 23) if big > 0 else 0.0
    bound = max(2.0 * err32, 4.0 * ulp)
    assert err <= bound, f'{what}: kernel error {err:.3e} vs float64 > {bound:.3e} (fp32 torch ops {err32:.3e}, 4 ulp {4 * ulp:.3e})'
