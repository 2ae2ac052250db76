"""Generates tests/golden/nll/*.npz: everything the UNMODIFIED reference ``forward(..., return_info=True)`` returns in eval
mode (ConditionalDDPM conditional_model.py:202, SimpleConditionalDDPM :727, EnVariationalDiffusion en_diffusion.py:336),
driven by the CPU denoiser stand-in with fixed torch seeds; the two T = 500 cases of nll_float64_cases.py additionally with
the timestep draw injected (t = 1, T and two interior steps in one batch).  They pin the likelihood evaluation of this repo
(noising, loss terms, KL prior, size prior, constants) independently of the CUDA kernels.  Needs the reference checkout
named by DIFFSBDD_REFERENCE."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from diffsbdd_b200 import synthetic as syn  # noqa: E402
from oracle import ref_shim  # noqa: E402
from ddpm_cases import DDPM_CFG, JOINT_CFG, OracleDynamics, make_pocket  # noqa: E402
from nll_cases import NLL_CASES, RETURN_NAMES, ddpm_kwargs, make_case_ligand  # noqa: E402
from nll_float64_cases import NLL_T500_CASES, T500_POCKET, T500_STEPS  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'nll')


def main():
    ref = ref_shim.load_reference()
    classes = {'conditional': ref.ConditionalDDPM, 'simple': ref.conditional_model.SimpleConditionalDDPM,
               'joint': ref.EnVariationalDiffusion}
    os.makedirs(OUT, exist_ok=True)
    for name, spec in {**NLL_CASES, **NLL_T500_CASES}.items():
        cfg, wseed = (JOINT_CFG, 6) if spec['model'] == 'joint' else (DDPM_CFG, 5)
        torch.manual_seed(0)                 # initialises the learned noise schedule; its weights are stored below
        ddpm = classes[spec['model']](dynamics=OracleDynamics(cfg, syn.synthetic_state_dict(cfg, wseed)), **ddpm_kwargs(spec))
        ddpm.eval()
        torch.manual_seed(spec['seed'])
        ligand, pocket, randint = make_case_ligand(spec), make_pocket(), torch.randint
        if name in NLL_T500_CASES:
            pocket = syn.synthetic_pocket(DDPM_CFG, T500_POCKET, seed=31, spread=3.0)
            torch.randint = lambda lo, hi, size, device=None: torch.tensor(T500_STEPS).view(size)
        try:
            out = ddpm(ligand, pocket, return_info=True)
        finally:
            torch.randint = randint
        arrays = {k: v.detach().numpy() for k, v in zip(RETURN_NAMES, out[:-1])}
        arrays.update({'info_' + k: v.detach().numpy() for k, v in out[-1].items()})
        arrays.update({'gamma.' + k: v.detach().numpy() for k, v in ddpm.gamma.state_dict().items()})
        np.savez_compressed(os.path.join(OUT, name + '.npz'), **arrays)
        print(name, {k: float(np.asarray(v).sum()) for k, v in arrays.items() if not k.startswith('gamma.')})


if __name__ == '__main__':
    main()
