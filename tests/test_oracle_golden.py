"""CPU: the travelling oracle (oracle/egnn_oracle.py) against the golden vectors that the UNMODIFIED
reference produced (tests/golden/make_golden.py)."""
import pytest
import torch

from helpers import golden_cases, load_golden, assert_close
from oracle import egnn_oracle


@pytest.mark.parametrize('case', golden_cases())
def test_oracle_matches_golden(case):
    cfg, sd, inp, want, edges = load_golden(case)
    got_a, got_r, got_edges = egnn_oracle.denoiser_forward(cfg, sd, *inp, return_edges=True)
    assert torch.equal(got_edges, edges), 'edge list differs from the reference get_edges'
    # same ATen ops in the same order: agreement is at the level of a few last bits, far inside the stated tolerance (the
    # host BLAS picks its kernels, and so its summation order, by CPU type: the goldens were written on another host)
    assert_close(got_a, want[0], 'ligand output', atol=5e-7, rtol=1e-6)
    assert_close(got_r, want[1], 'pocket output', atol=5e-7, rtol=1e-6)


@pytest.mark.parametrize('case', ['config1_n64_l4', 'joint_b2_h128_l5'])
def test_oracle_fp64_noise_floor(case):
    """fp32 oracle vs fp64 oracle: documents the reference's own rounding noise (SURVEY.md §4)."""
    cfg, sd, inp, want, _ = load_golden(case)
    o64 = egnn_oracle.denoiser_forward(cfg, sd, *inp, dtype=torch.float64)
    assert_close(want[0], o64[0], 'ligand fp32 vs fp64', atol=2e-6, rtol=1e-5)
    assert_close(want[1], o64[1], 'pocket fp32 vs fp64', atol=2e-6, rtol=1e-5)


def test_oracle_nan_convention():
    cfg, sd, inp, _, _ = load_golden('config1_n64_l4')
    bad = inp[0].clone()
    bad[0, 0] = float('nan')
    with pytest.raises(ValueError, match='NaN detected in EGNN output'):
        egnn_oracle.denoiser_forward(cfg, sd, bad, *inp[1:])
