"""CPU: the seeded-sampling contract that does not need a GPU — the numpy restatement of the generator against the
published Philox4x32-10 answers, argument validation of ``seeds=``, the seeded inverse-CDF size draw, and the shard
slicing of seeds."""
import numpy as np
import pytest
import torch

import seeded_cases as sc
from ddpm_cases import DDPM_CFG, HIST, make_pocket
from diffsbdd_b200 import seeded, synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM
from diffsbdd_b200.distributed import sample_given_pocket_sharded, shard_bounds, shard_seeds
from oracle.cpu_denoiser import OracleDynamics


# ---- generator restatement --------------------------------------------------------------------------------------------
# Known-answer vectors of Philox4x32-10 (Random123 kat_vectors: counter, key -> output)
KAT = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
       ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
       ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
        (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


@pytest.mark.parametrize('ctr,key,want', KAT)
def test_philox_known_answers(ctr, key, want):
    got = sc.philox4x32_10(*[np.array([c]) for c in ctr], np.array([key[0]]), np.array([key[1]]))
    assert [int(w[0]) for w in got] == list(want)


def test_counter_layout_is_per_graph():
    """A graph's words depend on its seed and its own rows only: the same graph at another batch position gives the same
    words; another seed or draw id changes them."""
    lig = np.repeat([0, 1, 2], [3, 5, 2])
    poc = np.repeat([0, 1, 2], [4, 6, 1])
    w = sc.words(sc.ROLE_JOINT_X, 3, [7, 11, 7], 5, lig, poc)
    alone = sc.words(sc.ROLE_JOINT_X, 3, [11], 5, np.zeros(5, int), np.zeros(6, int))
    rows_g1 = np.r_[3:8, 10 + 4:10 + 10]
    assert np.array_equal(w[rows_g1], alone)
    assert not np.array_equal(sc.words(sc.ROLE_LIGAND, 5, [11], 5, np.zeros(5, int), None), sc.words(
        sc.ROLE_LIGAND, 5, [12], 5, np.zeros(5, int), None))
    assert not np.array_equal(sc.words(sc.ROLE_LIGAND, 5, [11], 5, np.zeros(5, int), None), sc.words(
        sc.ROLE_LIGAND, 5, [11], 6, np.zeros(5, int), None))
    # graphs 0 and 2 share a seed and a layout prefix: their first ligand rows are equal
    assert np.array_equal(w[0:2], w[8:10])


def test_box_muller_restatement_moments():
    w = sc.words(sc.ROLE_LIGAND, 8, [2024], seeded.draw_id(1, 3, 0, 0), np.zeros(50000, int), None)
    z = sc.normals(w).ravel()
    assert abs(z.mean()) < 0.01 and abs(z.var() - 1) < 0.01
    u = sc.uniform(w)
    assert u.min() > 0 and u.max() <= 1


def test_draw_id_layout():
    assert seeded.draw_id(seeded.STAGE_LOOP, 499, 3, seeded.PURPOSE_RENOISE) == (1 << 40) | (499 << 20) | (3 << 4) | 2
    with pytest.raises(ValueError):
        seeded.draw_id(seeded.STAGE_LOOP, 1 << 20)


# ---- argument validation --------------------------------------------------------------------------------------------
@pytest.mark.parametrize('seeds,exc', [([1, 2, 3], ValueError), ([1.0, 2.0], TypeError), (torch.tensor([1.5, 2.0]), TypeError),
                                       ([-1, 2], ValueError), (np.array([2 ** 63, 1], dtype=np.uint64), ValueError),
                                       (torch.tensor([[1, 2]]), ValueError), (['a', 'b'], TypeError)])
def test_bad_seeds_are_rejected(seeds, exc):
    with pytest.raises(exc):
        seeded.host_seeds(seeds, 2)


def test_good_seeds_accepted():
    for s in ([0, 2 ** 63 - 1], np.array([3, 4], dtype=np.uint32), torch.tensor([5, 6], dtype=torch.int32), (7, 8)):
        out = seeded.host_seeds(s, 2)
        assert out.dtype == torch.int64 and out.shape == (2,) and out.tolist() == [int(v) for v in s]
    assert seeded.as_seeds(None, 2, 'cpu') is None


def _ddpm():
    sd = syn.synthetic_state_dict(DDPM_CFG, 5)
    return ConditionalDDPM(dynamics=OracleDynamics(DDPM_CFG, sd), atom_nf=DDPM_CFG.atom_nf, residue_nf=DDPM_CFG.residue_nf,
                           n_dims=3, timesteps=3, noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2',
                           norm_values=(1, 4), size_histogram=HIST).eval()


def test_cpu_run_with_seeds_raises():
    ddpm = _ddpm()
    with pytest.raises(RuntimeError, match='CUDA'):
        ddpm.sample_given_pocket(make_pocket('cpu'), torch.tensor([4, 3]), seeds=[1, 2])
    with pytest.raises(RuntimeError, match='CUDA'):
        ddpm.sample_given_pocket(make_pocket('cpu'), torch.tensor([4, 3]), seeds=torch.tensor([1, 2]))


# ---- size prior ---------------------------------------------------------------------------------------------------------
def test_inverse_cdf_matches_histogram():
    rng = np.random.default_rng(0)
    prob = torch.tensor(HIST).float() + 1e-3
    prob = prob / prob.sum()
    n_poc = rng.integers(0, prob.shape[1], size=4000)
    u = rng.random(4000).astype(np.float32) + np.float32(2 ** -33)
    got = seeded.inverse_cdf(prob, torch.from_numpy(n_poc), torch.from_numpy(u)).numpy()
    assert np.array_equal(got, sc.expected_sizes(prob.numpy(), n_poc, u))
    for j in range(prob.shape[1]):           # frequencies follow the conditional histogram column
        sel = got[n_poc == j]
        freq = np.bincount(sel, minlength=prob.shape[0]) / len(sel)
        want = (prob[:, j] / prob[:, j].sum()).numpy()
        assert np.abs(freq - want).max() < 4 * np.sqrt(0.25 / len(sel))
    # edges: u = 1 takes the last bin, u just above 0 the first non-empty one
    edge = seeded.inverse_cdf(prob, torch.tensor([0, 0]), torch.tensor([1.0, 2 ** -33])).tolist()
    assert edge == [prob.shape[0] - 1, 0]


# ---- sharding -------------------------------------------------------------------------------------------------------------
def test_shard_seeds_reassemble_the_job():
    seeds = torch.arange(100, 113)
    for w in (1, 2, 3, 8):
        parts = [shard_seeds(seeds, *shard_bounds(13, w, r)) for r in range(w)]
        assert torch.equal(torch.cat(parts), seeds)
    assert shard_seeds([5, 6, 7], 1, 3).tolist() == [6, 7]


class _Recorder:
    n_dims, atom_nf, residue_nf = 3, 2, 2

    def __init__(self):
        self.calls = []

    def sample_given_pocket(self, pocket, n_lig, timesteps=None, seeds=None):
        self.calls.append(seeds)
        n = int(n_lig.sum())
        return (torch.zeros((n, 5)), torch.zeros((len(pocket['x']), 5)), torch.zeros(n, dtype=torch.int64),
                pocket['mask'])


def test_sharded_call_passes_seed_slice_and_ignores_base_seed():
    pocket = syn.synthetic_pocket(DDPM_CFG, [4, 5, 6], seed=1, spread=2.0)
    state = torch.random.get_rng_state()
    rec = _Recorder()
    sample_given_pocket_sharded(rec, pocket, torch.tensor([2, 3, 1]), base_seed=999, seeds=[10, 20, 30])
    assert rec.calls[0].tolist() == [10, 20, 30]
    assert torch.equal(torch.random.get_rng_state(), state)
    with pytest.raises(ValueError):
        sample_given_pocket_sharded(rec, pocket, torch.tensor([2, 3, 1]), seeds=[10, 20])
    rec.calls.clear()
    sample_given_pocket_sharded(rec, pocket, torch.tensor([2, 3, 1]))      # unseeded: no seeds argument reaches the sampler
    assert rec.calls == [None]


def test_schedule_must_fit_the_draw_id():
    seeded.check_schedule(1 << 20, 1 << 16)
    with pytest.raises(ValueError):
        seeded.check_schedule((1 << 20) + 1)
    with pytest.raises(ValueError):
        seeded.check_schedule(500, (1 << 16) + 1)
    # the joint model's rounds are its RePaint blocks: resamplings x T / jump_length of them
    from diffsbdd_b200.en_diffusion import EnVariationalDiffusion
    blocks = len(EnVariationalDiffusion.get_repaint_schedule(200, 1, 400))
    assert blocks > 1 << 16
    with pytest.raises(ValueError):
        seeded.check_schedule(400, blocks)
