"""CPU: the C-ABI library builds for sm_90a, loads, exports every symbol include/diffsbdd_b200.h declares, and its
host-side logic (parameter table, config validation, size helpers) behaves — no compute calls (no GPU here)."""
import ctypes as C
import os
import re

import pytest

from diffsbdd_b200 import _build, _native, synthetic as syn
from diffsbdd_b200.config import DynamicsConfig, FULLATOM_COND, CA_COND
from diffsbdd_b200.dynamics import EGNNDynamics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    _build.build()
    return _native.load(build_if_missing=False)


def header_symbols():
    text = open(os.path.join(ROOT, 'include', 'diffsbdd_b200.h')).read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(dsb_[a-z_0-9]+)\s*\(', text)))


def test_header_symbols_all_exported(lib):
    syms = header_symbols()
    assert len(syms) >= 12
    for s in syms:
        assert hasattr(lib, s), f'{s} declared in include/diffsbdd_b200.h but not exported'
    assert sorted(_native.EXPORTED_SYMBOLS) == syms


def test_library_is_sm90a_only(lib):
    out = os.popen(f'cuobjdump -lelf {_native.lib_path()} 2>/dev/null').read()
    if out.strip():
        assert 'sm_90a' in out and not re.search(r'sm_(?!90a)\d+', out), out


@pytest.mark.parametrize('cfg', [FULLATOM_COND, CA_COND,
                                 DynamicsConfig(hidden_nf=192, edge_embedding_dim=8, n_layers=3),
                                 DynamicsConfig(reflection_equivariant=True, inv_sublayers=2, attention=False, hidden_nf=128)])
def test_param_table_matches_reference_state_dict_layout(lib, cfg):
    net = EGNNDynamics.from_config(cfg)
    got = _native.param_names(net._c_config())
    want = [(k, 1) for k, shape, _ in syn.state_dict_spec(cfg)]
    assert [g[0] for g in got] == [w[0] for w in want]
    sd = net.state_dict()
    for name, numel in got:
        assert sd[name].numel() == numel, name
    extra = set(sd) - {g[0] for g in got}
    assert all(k.endswith('cross_product_mlp.4.weight') for k in extra)     # the aliased shared layer


def test_invalid_configs_are_rejected_with_messages(lib):
    net = EGNNDynamics.from_config(FULLATOM_COND)
    c = net._c_config()
    c.hidden_nf = 100
    assert lib.dsb_param_count(C.byref(c)) == -2
    assert b'hidden_nf' in lib.dsb_last_error()
    c = net._c_config(); c.n_dims = 2
    assert lib.dsb_param_count(C.byref(c)) == -2
    c = net._c_config(); c.normalization_factor = 0.0
    assert lib.dsb_param_count(C.byref(c)) == -1
    out = C.c_void_p()
    assert lib.dsb_dynamics_create(C.byref(net._c_config()), None, 0, C.byref(out)) == -1
    assert out.value is None


def test_edge_capacity_helper(lib):
    nl = (C.c_int64 * 3)(25, 1, 0)
    npk = (C.c_int64 * 3)(175, 9, 4)
    assert lib.dsb_edge_capacity(nl, npk, 3) == 200 * 200 + 100 + 16


def test_unsupported_reference_options_fail_loudly():
    sin = EGNNDynamics(10, 10, 3, sin_embedding=True, hidden_nf=128)       # built since round 2 (fp32 FFMA kernels only)
    assert sin.cfg.sin_embedding and sin.math_mode == 0
    assert dict(sin.named_parameters())['egnn.e_block_0.gcl_0.edge_mlp.0.weight'].shape == (128, 2 * 128 + 24)
    assert EGNNDynamics(10, 10, 3, aggregation_method='mean').cfg.aggregation_method == 'mean'     # built since round 2
    with pytest.raises(ValueError):
        EGNNDynamics(10, 10, 3, aggregation_method='max')
    with pytest.raises(NotImplementedError):
        EGNNDynamics(10, 10, 3, mode='gnn_dynamics')
    with pytest.raises(Exception, match='Wrong mode'):
        EGNNDynamics(10, 10, 3, mode='nonsense')


def test_no_cpu_fallback():
    import torch
    net = EGNNDynamics.from_config(FULLATOM_COND.with_(n_layers=1, hidden_nf=64)).eval()
    inp = syn.synthetic_denoiser_inputs(net.cfg, [3], [5], seed=0)
    with torch.no_grad(), pytest.raises(RuntimeError, match='no CPU fallback'):
        net(*inp)
