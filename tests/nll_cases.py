"""Shared definitions of the likelihood-evaluation (eval-mode ``forward``) cases: golden generator and tests."""
import torch

from ddpm_cases import DDPM_CFG, JOINT_CFG, make_ligand, make_pocket  # noqa: F401

# joint size histogram covering the ligand sizes below and the pockets of make_pocket() (22 and 17 nodes)
NLL_HIST = [[float((3 * i + 5 * j) % 7) + 0.5 for j in range(26)] for i in range(12)]

RETURN_NAMES = ('delta_log_px', 'error_t_lig', 'error_t_pocket', 'SNR_weight', 'loss_0_x_ligand', 'loss_0_x_pocket',
                'loss_0_h', 'neg_log_constants', 'kl_prior', 'log_pN', 't_int', 'xh_lig_hat')

VNODE = DDPM_CFG.atom_nf - 1

NLL_CASES = {
    'cond_ragged': dict(model='conditional', n_lig=[7, 5], T=20, schedule='polynomial_2', seed=301),
    'cond_simple': dict(model='simple', n_lig=[4, 9], T=20, schedule='polynomial_2', seed=302),
    'joint': dict(model='joint', n_lig=[6, 4], T=20, schedule='polynomial_2', seed=303),
    'cond_vnode': dict(model='conditional', n_lig=[8, 6], T=20, schedule='polynomial_2', seed=304, vnode=True),
    'cond_learned': dict(model='conditional', n_lig=[5, 3], T=50, schedule='learned', seed=305),
}


def make_case_ligand(spec, device='cpu'):
    """Ligand dict of a case; with ``vnode`` the last two atoms of every graph are virtual (one-hot class VNODE)."""
    lig, _ = make_ligand(spec['n_lig'], 0, device=device)
    if spec.get('vnode'):
        ends = torch.cumsum(torch.tensor(spec['n_lig']), 0)
        rows = torch.cat([torch.arange(e - 2, e) for e in ends.tolist()]).to(device)
        lig['one_hot'][rows] = 0
        lig['one_hot'][rows, VNODE] = 1
    return lig


def ddpm_kwargs(spec):
    cfg = JOINT_CFG if spec['model'] == 'joint' else DDPM_CFG
    return dict(atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=spec['T'],
                noise_schedule=spec['schedule'], noise_precision=5e-4, loss_type='vlb', norm_values=(1, 4),
                size_histogram=NLL_HIST, virtual_node_idx=VNODE if spec.get('vnode') else None)
