"""Generates tests/golden/ddpm/*.npz: outputs of the UNMODIFIED reference ``ConditionalDDPM`` samplers
(conditional_model.py:479, :558, :364) driven by a CPU denoiser stand-in (the oracle restatement of
EGNNDynamics.forward, bit-identical to the reference module on CPU — tests/test_oracle_golden.py), with
fixed torch seeds.  They pin the DDPM wrapper of this repo (schedule, mu/sigma update, COM handling,
RePaint loop) independently of the CUDA kernels.  Needs the reference checkout named by DIFFSBDD_REFERENCE."""
from __future__ import annotations

import copy
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from diffsbdd_b200 import synthetic as syn  # noqa: E402
from oracle import ref_shim  # noqa: E402
from ddpm_cases import (DDPM_CFG, HIST, OracleDynamics, make_pocket, make_ligand, SAMPLER_CASES,  # noqa: E402
                        JOINT_CFG, JOINT_CASES, make_pocket_fixed)

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'ddpm')


def main():
    ref = ref_shim.load_reference()
    sd = syn.synthetic_state_dict(DDPM_CFG, 5)
    for name, spec in SAMPLER_CASES.items():
        dyn = OracleDynamics(DDPM_CFG, sd)
        ddpm = ref.ConditionalDDPM(dynamics=dyn, atom_nf=DDPM_CFG.atom_nf, residue_nf=DDPM_CFG.residue_nf,
                                   n_dims=3, timesteps=spec['T'], noise_schedule='polynomial_2',
                                   noise_precision=5e-4, loss_type='l2', norm_values=(1, 4), size_histogram=HIST)
        ddpm.eval()
        pocket = make_pocket()
        torch.manual_seed(spec['seed'])
        if spec['kind'] == 'sample':
            out = ddpm.sample_given_pocket(pocket, torch.tensor(spec['n_lig']), return_frames=spec['frames'],
                                           timesteps=spec['timesteps'])
        elif spec['kind'] == 'inpaint':
            lig, fixed = make_ligand(spec['n_lig'], spec['n_fixed'])
            out = ddpm.inpaint(lig, pocket, fixed, resamplings=spec['resamplings'], timesteps=spec['timesteps'],
                               center=spec['center'])
        else:
            lig, _ = make_ligand(spec['n_lig'], 0)
            out = ddpm.diversify(lig, pocket, noising_steps=spec['noising_steps'])
        np.savez_compressed(os.path.join(OUT, name + '.npz'), xh_lig=out[0].numpy(), xh_pocket=out[1].numpy(),
                            lig_mask=out[2].numpy(), pocket_mask=out[3].numpy(),
                            gamma=ddpm.gamma.gamma.detach().numpy())
        print(name, tuple(out[0].shape), float(out[0].abs().max()))
    # joint model: the UNMODIFIED reference EnVariationalDiffusion (en_diffusion.py:677, :839)
    sdj = syn.synthetic_state_dict(JOINT_CFG, 6)
    for name, spec in JOINT_CASES.items():
        ddpm = ref.EnVariationalDiffusion(dynamics=OracleDynamics(JOINT_CFG, sdj), atom_nf=JOINT_CFG.atom_nf,
                                          residue_nf=JOINT_CFG.residue_nf, n_dims=3, timesteps=spec['T'],
                                          noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2',
                                          norm_values=(1, 4), size_histogram=HIST)
        ddpm.eval()
        pocket = make_pocket()
        torch.manual_seed(spec['seed'])
        if spec['kind'] == 'sample':
            out = ddpm.sample(len(spec['n_lig']), torch.tensor(spec['n_lig']), pocket['size'],
                              return_frames=spec['frames'], timesteps=spec['timesteps'])
        else:
            lig, fixed = make_ligand(spec['n_lig'], spec['n_fixed'])
            out = ddpm.inpaint(lig, pocket, fixed, make_pocket_fixed(spec, pocket), resamplings=spec['resamplings'],
                               jump_length=spec['jump_length'], return_frames=spec['frames'],
                               timesteps=spec['timesteps'])
        np.savez_compressed(os.path.join(OUT, name + '.npz'), xh_lig=out[0].numpy(), xh_pocket=out[1].numpy(),
                            lig_mask=out[2].numpy(), pocket_mask=out[3].numpy(),
                            gamma=ddpm.gamma.gamma.detach().numpy())
        print(name, tuple(out[0].shape), float(out[0].abs().max()))


if __name__ == '__main__':
    main()
