"""CPU: plumbing of the deterministic mode — the C ABI entry point, the Python setting ('auto' / True / False, the
DSB_DETERMINISTIC environment variable), the capture signature, and the CPU path of the scatter stand-ins (unchanged)."""
import ctypes as C

import pytest
import torch

from diffsbdd_b200 import _build, _native
from diffsbdd_b200.config import DynamicsConfig
from diffsbdd_b200.dynamics import EGNNDynamics
from diffsbdd_b200.en_diffusion import deterministic_reductions, scatter_add, scatter_mean

CFG = DynamicsConfig(joint_nf=16, hidden_nf=64, n_layers=2)


@pytest.fixture(scope='module')
def lib():
    _build.build()
    return _native.load(build_if_missing=False)


def test_set_deterministic_exported_and_rejects_null(lib):
    assert 'dsb_dynamics_set_deterministic' in _native.EXPORTED_SYMBOLS
    assert lib.dsb_dynamics_set_deterministic(C.c_void_p(None), 1) == -1      # DSB_ERR_INVALID_ARGUMENT
    assert lib.dsb_dynamics_set_deterministic(C.c_void_p(None), -1) == -1
    assert 'null' in lib.dsb_last_error().decode()


def test_auto_follows_torch_switch(monkeypatch):
    monkeypatch.delenv('DSB_DETERMINISTIC', raising=False)
    net = EGNNDynamics.from_config(CFG)
    assert net.deterministic == 'auto'
    prev = torch.are_deterministic_algorithms_enabled()
    prev_warn = torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        torch.use_deterministic_algorithms(True, warn_only=True)
        assert net.deterministic_active is True
        torch.use_deterministic_algorithms(False)
        assert net.deterministic_active is False
        net.deterministic = True
        assert net.deterministic_active is True
        torch.use_deterministic_algorithms(True, warn_only=True)
        net.deterministic = False
        assert net.deterministic_active is False
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


@pytest.mark.parametrize('env,want', [('1', True), ('0', False), ('auto', 'auto'), ('true', True), ('off', False)])
def test_environment_variable_sets_initial_mode(monkeypatch, env, want):
    monkeypatch.setenv('DSB_DETERMINISTIC', env)
    assert EGNNDynamics.from_config(CFG).deterministic == want


def test_bad_setting_rejected(monkeypatch):
    monkeypatch.setenv('DSB_DETERMINISTIC', 'sometimes')
    with pytest.raises(ValueError):
        EGNNDynamics.from_config(CFG)
    monkeypatch.delenv('DSB_DETERMINISTIC')
    net = EGNNDynamics.from_config(CFG)
    with pytest.raises(ValueError):
        net.deterministic = 'maybe'


def test_state_dict_and_constructor_unchanged(monkeypatch):
    monkeypatch.setenv('DSB_DETERMINISTIC', '1')
    a = EGNNDynamics.from_config(CFG)
    monkeypatch.setenv('DSB_DETERMINISTIC', '0')
    b = EGNNDynamics.from_config(CFG)
    assert list(a.state_dict()) == list(b.state_dict())
    b.load_state_dict(a.state_dict())


def test_capture_signature_differs_between_modes(lib, monkeypatch):
    monkeypatch.delenv('DSB_DETERMINISTIC', raising=False)
    net = EGNNDynamics.from_config(CFG)
    net.deterministic = False
    off = net.capture_signature()
    net.deterministic = True
    on = net.capture_signature()
    assert off != on
    net.deterministic = 'auto'
    prev = torch.are_deterministic_algorithms_enabled()
    prev_warn = torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        torch.use_deterministic_algorithms(True, warn_only=True)
        assert net.capture_signature() == on
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
    assert net.capture_signature() == (off if not prev else on)


def test_cpu_scatter_unchanged_inside_deterministic_reductions():
    g = torch.Generator().manual_seed(0)
    src = torch.randn(37, 3, generator=g)
    idx = torch.repeat_interleave(torch.arange(5), torch.tensor([9, 0, 11, 7, 10]))
    want_add, want_mean = scatter_add(src, idx), scatter_mean(src, idx, dim_size=6)
    with deterministic_reductions(True):
        assert torch.equal(scatter_add(src, idx), want_add)
        assert torch.equal(scatter_mean(src, idx, dim_size=6), want_mean)
    want = torch.zeros(5, 3, dtype=torch.float64).index_add_(0, idx, src.double())
    assert torch.allclose(want_add.double(), want, atol=1e-6)
