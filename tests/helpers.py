"""Shared helpers for the parity tests."""
import glob
import json
import os

import numpy as np
import torch

from diffsbdd_b200.config import CONFIG1, DynamicsConfig
from diffsbdd_b200 import synthetic as syn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
# stated fp32 parity tolerance for one denoiser forward (SURVEY.md §4: ~20x the reference's own
# fp32-vs-fp64 noise floor of 3-4e-7, far below TF32's ~1e-3)
ATOL, RTOL = 1e-5, 1e-4

# configurations whose reference state-dict layout (keys in order, shapes) is stored in golden/layout/reference_state_dict_layout.npz
# (golden/make_layout_golden.py): one string array per configuration, entries "<key>:<d0>x<d1>..."
LAYOUT_CASES = {
    'config1': CONFIG1,
    'update_pocket_reflect_h128': DynamicsConfig(update_pocket_coords=True, reflection_equivariant=True, hidden_nf=128),
    'emb8_h192_l2_noatt': DynamicsConfig(edge_embedding_dim=8, hidden_nf=192, n_layers=2, attention=False),
}


def reference_state_dict_layout(name):
    entries = np.load(os.path.join(GOLDEN, 'layout', 'reference_state_dict_layout.npz'), allow_pickle=False)[name]
    out = []
    for e in entries.tolist():
        k, shape = e.rsplit(':', 1)
        out.append((k, tuple(int(d) for d in shape.split('x')) if shape else ()))
    return out


def golden_cases():
    return sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN, '*.npz')))


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, name + '.npz'), allow_pickle=False)
    cfg = DynamicsConfig(**json.loads(str(z['cfg'])))
    sd = syn.synthetic_state_dict(cfg, int(z['weight_seed']))
    chk = syn.state_dict_checksum(sd)
    assert abs(chk - float(z['weight_checksum'])) <= 1e-9 * max(1.0, abs(chk)), 'weight recipe drifted'
    inp = (torch.from_numpy(z['xh_atoms']), torch.from_numpy(z['xh_residues']), torch.from_numpy(z['t']),
           torch.from_numpy(z['mask_atoms']), torch.from_numpy(z['mask_residues']))
    out = (torch.from_numpy(z['out_atoms']), torch.from_numpy(z['out_residues']))
    edges = torch.from_numpy(z['edges'].astype(np.int64))
    return cfg, sd, inp, out, edges


def assert_close(got, want, what, atol=ATOL, rtol=RTOL):
    got, want = got.detach().cpu().double(), want.detach().cpu().double()
    assert got.shape == want.shape, (what, got.shape, want.shape)
    err = (got - want).abs()
    tol = atol + rtol * want.abs()
    worst = float((err - tol).max()) if err.numel() else -1.0
    assert worst <= 0, f'{what}: max abs err {float(err.max()):.3e} exceeds atol={atol} rtol={rtol}'
    return float(err.max()) if err.numel() else 0.0
