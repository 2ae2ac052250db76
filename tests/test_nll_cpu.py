"""CPU: the eval-mode likelihood ``forward`` of this repo's DDPM classes (eager engine, oracle denoiser) reproduces what the
UNMODIFIED reference returned (tests/golden/nll/*.npz, tests/golden/make_golden_nll.py) under the same torch seed."""
import math
import os

import numpy as np
import pytest
import torch

from ddpm_cases import DDPM_CFG, JOINT_CFG, OracleDynamics, make_pocket
from nll_cases import NLL_CASES, NLL_HIST, RETURN_NAMES, ddpm_kwargs, make_case_ligand
from diffsbdd_b200 import synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM, SimpleConditionalDDPM
from diffsbdd_b200.en_diffusion import DistributionNodes, EnVariationalDiffusion

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'nll')
CLASSES = {'conditional': ConditionalDDPM, 'simple': SimpleConditionalDDPM, 'joint': EnVariationalDiffusion}


def build_case(spec, gold=None, device='cpu'):
    cfg, wseed = (JOINT_CFG, 6) if spec['model'] == 'joint' else (DDPM_CFG, 5)
    ddpm = CLASSES[spec['model']](dynamics=OracleDynamics(cfg, syn.synthetic_state_dict(cfg, wseed), device=device),
                                  **ddpm_kwargs(spec))
    if gold is not None:
        ddpm.gamma.load_state_dict({k[len('gamma.'):]: torch.from_numpy(gold[k]) for k in gold.files if k.startswith('gamma.')})
    ddpm.loop_engine = 'eager'
    return ddpm.to(device).eval()


@pytest.mark.parametrize('name', sorted(NLL_CASES))
def test_forward_matches_reference_golden(name):
    spec = NLL_CASES[name]
    gold = np.load(os.path.join(GOLD, name + '.npz'))
    ddpm = build_case(spec, gold)
    torch.manual_seed(spec['seed'])
    out = ddpm(make_case_ligand(spec), make_pocket(), return_info=True)
    assert len(out) == len(RETURN_NAMES) + 1
    for key, got in zip(RETURN_NAMES, out[:-1]):
        want = torch.from_numpy(gold[key])
        assert tuple(got.shape) == tuple(want.shape), key
        assert torch.allclose(got.float(), want.float(), atol=1e-5, rtol=1e-5), (key, got, want)
    info = out[-1]
    assert sorted('info_' + k for k in info) == sorted(k for k in gold.files if k.startswith('info_'))
    for k, v in info.items():
        assert torch.allclose(v, torch.from_numpy(gold['info_' + k]), atol=1e-5, rtol=1e-5), k


def test_conditional_terms_are_consistent():
    """Seed-independent structure: t in [1, T], negative SNR weight, non-negative KL prior, zero pocket terms."""
    spec = NLL_CASES['cond_ragged']
    ddpm = build_case(spec)
    torch.manual_seed(0)
    out = ddpm(make_case_ligand(spec), make_pocket())
    t_int, snr = out[10], out[3]
    assert torch.all((t_int >= 1) & (t_int <= spec['T']))
    assert torch.all(snr < 0)
    assert torch.all(out[8] >= -1e-6)
    assert float(out[2]) == 0.0 and float(out[5]) == 0.0
    assert out[11].shape == (sum(spec['n_lig']), 3 + DDPM_CFG.atom_nf)


def test_distribution_nodes_log_prob_matches_histogram():
    dist = DistributionNodes(NLL_HIST)
    hist = np.asarray(NLL_HIST, dtype=np.float64) + 1e-3
    p = hist / hist.sum()
    n1, n2 = torch.tensor([0, 3, 11, 7]), torch.tensor([25, 0, 4, 17])
    got = dist.log_prob(n1, n2)
    want = [math.log(p[a, b]) for a, b in zip(n1.tolist(), n2.tolist())]
    assert np.allclose(got.numpy(), want, atol=1e-5)
    # the conditional prior is the same table normalised over the ligand axis
    cond = dist.log_prob_n1_given_n2(n1, n2)
    want_c = [math.log(p[a, b] / p[:, b].sum()) for a, b in zip(n1.tolist(), n2.tolist())]
    assert np.allclose(cond.numpy(), want_c, atol=1e-5)


@pytest.mark.parametrize('model', sorted(CLASSES))
def test_forward_raises_in_training_mode(model):
    spec = dict(NLL_CASES['joint' if model == 'joint' else 'cond_ragged'], model=model)
    ddpm = build_case(spec).train()
    with pytest.raises(NotImplementedError):
        ddpm(make_case_ligand(spec), make_pocket())
