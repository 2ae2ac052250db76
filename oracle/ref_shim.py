"""TEST INFRASTRUCTURE ONLY — imports the *unmodified* reference from the checkout named by the environment
variable DIFFSBDD_REFERENCE.

Used by the generators under ``tests/golden/`` to produce the committed golden data; the tests themselves only
read that data and never need the reference.

The reference's DDPM wrapper imports ``torch_scatter`` and its top-level ``utils`` imports
``rdkit``/``Bio``/``networkx`` at module level (reference utils.py:6-9, en_diffusion.py:8); none is
installed here. The stubs below are registered in ``sys.modules`` *before* the import. They touch
nothing on the EGNN path (which uses ``Tensor.scatter_add_``, egnn_new.py:326) — only the COM
bookkeeping of the DDPM wrapper uses ``scatter_mean/scatter_add`` whose semantics (torch-scatter
2.0.9, README.md:60: output length ``index.max()+1`` unless ``dim_size``; mean = sum/count.clamp(1))
are restated here with ``index_add_``.
"""
from __future__ import annotations

import os
import sys
import types

import torch

REFERENCE_ROOT = os.environ.get('DIFFSBDD_REFERENCE', '')


def reference_available() -> bool:
    return bool(REFERENCE_ROOT) and os.path.isfile(os.path.join(REFERENCE_ROOT, 'equivariant_diffusion', 'egnn_new.py'))


def _scatter_add(src, index, dim=0, out=None, dim_size=None):
    assert dim == 0
    n = int(index.max()) + 1 if dim_size is None else dim_size
    res = torch.zeros((n,) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    return res.index_add_(0, index, src)


def _scatter_mean(src, index, dim=0, out=None, dim_size=None):
    s = _scatter_add(src, index, dim, None, dim_size)
    cnt = torch.zeros((s.shape[0],), dtype=src.dtype, device=src.device)
    cnt.index_add_(0, index, torch.ones_like(index, dtype=src.dtype))
    cnt = cnt.clamp(min=1)
    return s / cnt.view((-1,) + (1,) * (s.dim() - 1))


def _install_stubs():
    if 'torch_scatter' not in sys.modules:
        m = types.ModuleType('torch_scatter')
        m.scatter_add = _scatter_add
        m.scatter_mean = _scatter_mean
        sys.modules['torch_scatter'] = m
    for name in ('rdkit', 'rdkit.Chem', 'Bio', 'Bio.PDB', 'Bio.PDB.Polypeptide', 'networkx'):
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                sys.modules[name] = types.ModuleType(name)
    sys.modules['rdkit'].Chem = sys.modules['rdkit.Chem']
    sys.modules['Bio'].PDB = sys.modules['Bio.PDB']
    if not hasattr(sys.modules['Bio.PDB.Polypeptide'], 'is_aa'):
        sys.modules['Bio.PDB.Polypeptide'].is_aa = lambda *a, **k: True


def load_reference():
    """Returns a namespace with the reference's own classes (EGNNDynamics, ConditionalDDPM, ...)."""
    if not reference_available():
        raise RuntimeError(f'reference not found (DIFFSBDD_REFERENCE={REFERENCE_ROOT!r})')
    _install_stubs()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    from equivariant_diffusion import egnn_new, dynamics, en_diffusion, conditional_model
    ns = types.SimpleNamespace(
        egnn_new=egnn_new, dynamics=dynamics, en_diffusion=en_diffusion,
        conditional_model=conditional_model,
        EGNNDynamics=dynamics.EGNNDynamics,
        EnVariationalDiffusion=en_diffusion.EnVariationalDiffusion,
        ConditionalDDPM=conditional_model.ConditionalDDPM,
    )
    return ns


def build_reference_dynamics(cfg, state_dict):
    """Unmodified reference ``EGNNDynamics`` (dynamics.py:10) carrying the given weights, eval mode."""
    ref = load_reference()
    kw = cfg.kwargs()
    net = ref.EGNNDynamics(device='cpu', act_fn=torch.nn.SiLU(), **kw)
    missing, unexpected = net.load_state_dict(state_dict, strict=True), None
    net.eval()
    return net
