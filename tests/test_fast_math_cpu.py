"""CPU: the single-product FP16 math mode ('1xfp16') — its name and mask, and the error model the GPU per-launch checks
hold it to (fast_math_cases.Arith1x), checked against a float64 hand computation of the kernel's arithmetic."""
import math

import pytest
import torch

import fast_math_cases as fm
import launch_cases as lc
from diffsbdd_b200.config import DynamicsConfig
from diffsbdd_b200.dynamics import EGNNDynamics


@pytest.mark.parametrize('name,mask', [('1xfp16', 31), ('3xfp16', 15), ('3xtf32', 7), ('fp32', 0)])
def test_names_and_masks(name, mask):
    net = EGNNDynamics.from_config(DynamicsConfig(joint_nf=16, hidden_nf=128, n_layers=1))
    net.math_mode = name
    assert net.math_mode == mask


def test_environment_variable(monkeypatch):
    monkeypatch.setenv('DSB_MATH_MODE', '1xfp16')
    assert EGNNDynamics.from_config(DynamicsConfig(joint_nf=16, hidden_nf=256, n_layers=1)).math_mode == 31
    monkeypatch.setenv('DSB_MATH_MODE', '31')
    assert EGNNDynamics.from_config(DynamicsConfig(joint_nf=16, hidden_nf=256, n_layers=1)).math_mode == 31


@pytest.mark.parametrize('hidden,want', [(128, 15), (192, 15), (256, 15), (64, 0)])
def test_auto_unchanged(monkeypatch, hidden, want):
    monkeypatch.delenv('DSB_MATH_MODE', raising=False)
    assert EGNNDynamics.from_config(DynamicsConfig(joint_nf=16, hidden_nf=hidden, n_layers=1)).math_mode == want


# ---- the error model --------------------------------------------------------------------------------------------------
def _to_f32_toward_zero(x):
    """float64 -> the fp32 value next to x on the side of zero (a truncating accumulator)."""
    r = x.to(torch.float32)
    over = r.double().abs() > x.abs()
    return torch.where(over, torch.nextafter(r, torch.zeros_like(r)), r)


def kernel_single_product(a, W, b):
    """Hand computation of what the 1xFP16 kernel computes for a @ W^T + b, in float64: activations rounded to fp16,
    weights scaled by the image's power of two and rounded to fp16, exact products (11 x 11 bits), one truncating fp32
    accumulation per k-group of 16, then the epilogue fma acc * (1 / s) + b rounded to fp32."""
    s = fm.weight_scale(W)
    ah = a.to(torch.float32).to(torch.float16).double()
    wh = (W.to(torch.float32) * s).to(torch.float16).double()
    acc = torch.zeros(a.shape[0], W.shape[0], dtype=torch.float64)
    for k0 in range(0, a.shape[1], 16):
        acc = _to_f32_toward_zero(acc + ah[:, k0:k0 + 16] @ wh[:, k0:k0 + 16].T).double()
    return (acc / s + b.double()).to(torch.float32).double()


def _case(seed, K, spread):
    """Activations and weights whose magnitudes spread over 2^-spread .. 1 (spread 30 reaches fp16's subnormals)."""
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(24, K, generator=g, dtype=torch.float64) * 2.0 ** -(torch.rand(24, K, generator=g) * spread).floor()
    W = torch.randn(20, K, generator=g, dtype=torch.float64) * 2.0 ** -(torch.rand(20, K, generator=g) * spread).floor()
    b = torch.randn(20, generator=g, dtype=torch.float64) * 0.1
    return a.float().double(), W.float().double(), b.float().double()


@pytest.mark.parametrize('K', [16, 64, 256, 512])
@pytest.mark.parametrize('spread', [0, 8, 30])
def test_error_model_bounds_hand_computation(K, spread):
    worst = 0.0
    for seed in range(4):
        a, W, b = _case(seed, K, spread)
        got = kernel_single_product(a, W, b)
        exact = a @ W.T + b
        ar = fm.Arith1x(True)
        Wa, aa = W.abs(), a.abs()
        bound = ar.coef(K) * (aa @ Wa.T + b.abs()) + ar.floor(aa, Wa, float(Wa.max()))
        r = (got - exact).abs() / bound
        worst = max(worst, float(r.max()))
    assert worst <= 1.0, f'hand computation exceeds the single-product bound: {worst:.3f}'
    assert worst >= 0.02, f'bound is loose by more than 50x: {worst:.4f}'


def test_rounded_evaluation_rounds_as_the_kernel():
    """The float64 evaluation of the statistical criterion (fast_math_cases.contract) differs from the hand computation of
    the kernel only by the kernel's fp32 accumulation and epilogue."""
    a, W, b = _case(11, 256, 8)
    got = kernel_single_product(a, W, b)
    ref = fm.contract(a, W, b)
    M = fm.f16_act(a).abs() @ fm.f16_weight(W).abs().T + b.abs()
    acc_bound = (2 * math.ceil(256 / 16) * 17 * lc.U * 1.01 + 2 * lc.U) * M
    assert bool(((got - ref).abs() <= acc_bound).all())
    assert float((got - ref).abs().max()) < 0.05 * float((got - a @ W.T - b).abs().max())


def test_weight_scale_rule():
    for amax in (1e-6, 0.013, 0.5, 1.0, 3.7, 4096.0, 1e4):
        W = torch.tensor([[amax, -amax / 3]], dtype=torch.float64)
        s = fm.weight_scale(W)
        assert 4096.0 <= amax * s < 8192.0 and math.log2(s) == round(math.log2(s))
    assert fm.weight_scale(torch.zeros(2, 2)) == 1.0
