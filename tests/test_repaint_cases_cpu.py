"""CPU: the RePaint references and schedules of tests/repaint_cases.py.

* inpaint_update_ref / joint_inpaint_update_ref in fp32 reproduce, bit for bit, the eager samplers' RePaint iterations
  (ConditionalDDPM.inpaint, EnVariationalDiffusion.inpaint with jumps) run on the CPU around the oracle denoiser with a
  recorded noise tape.
* The replay schedules agree with the draw ids the eager loops set (``_draw_at``) for every run of the GPU trajectory
  tests and at the edges of get_repaint_schedule (a final partial block; jump_length dividing T or not), and no draw id
  repeats within a run.
* The step tables the graph engines read (_schedule_tables, the clamped t_back column of _joint_tables) agree with the
  eager loops' coefficient ops at every row.
"""
import pytest
import torch

import repaint_cases as rc
from ddpm_cases import DDPM_CFG, HIST, JOINT_CFG, make_ligand, make_pocket
from oracle.cpu_denoiser import OracleDynamics
from diffsbdd_b200 import seeded, synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion, scatter_mean

T = 500


def _ddpm(joint, T, dyn):
    cls = EnVariationalDiffusion if joint else ConditionalDDPM
    cfg = JOINT_CFG if joint else DDPM_CFG
    return cls(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=T,
               noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2', norm_values=(1, 4),
               size_histogram=HIST).eval()


def _oracle_ddpm(joint, T, weight_seed=5):
    cfg = JOINT_CFG if joint else DDPM_CFG
    return _ddpm(joint, T, OracleDynamics(cfg, syn.synthetic_state_dict(cfg, weight_seed)))


class _ZeroDynamics(torch.nn.Module):
    """A denoiser predicting zero noise: the eager loops' draw order does not depend on the denoiser."""

    def __init__(self, joint):
        super().__init__()
        self.update_pocket_coords = joint

    def forward(self, xh_lig, xh_pocket, t, lm, pm):
        return torch.zeros_like(xh_lig), torch.zeros_like(xh_pocket)


class _Tape:
    """Noise for the eager CPU loops from a seeded generator, every draw kept in order: ``sample_gaussian`` and the raw
    position draw of ``sample_center_gravity_zero_gaussian_batch`` (the joint model's COM-free noise)."""

    def __init__(self, ddpm, seed):
        self.g, self.draws = torch.Generator().manual_seed(seed), []
        ddpm.sample_gaussian = self.normal

        def centred(size, lig, pocket):
            x = self.normal(size, lig.device)
            return EnVariationalDiffusion.remove_mean_batch(x, torch.cat((lig, pocket)))
        ddpm.sample_center_gravity_zero_gaussian_batch = centred

    def normal(self, size, device):
        x = torch.randn(size, generator=self.g)
        self.draws.append(x.clone())
        return x.to(device)


def _record_reverse_calls(ddpm):
    """Keeps the input and output of every sample_p_zs_given_zt call and the input of sample_p_xh_given_z0."""
    calls, final = [], []
    orig, orig_final = ddpm.sample_p_zs_given_zt, ddpm.sample_p_xh_given_z0

    def step(s, t, zl, zp, lm, pm, fix_noise=False):
        out = orig(s, t, zl, zp, lm, pm, fix_noise)
        calls.append(((zl.clone(), zp.clone()), tuple(o.clone() for o in out)))
        return out

    def last(zl, zp, *args, **kw):
        final.append((zl.clone(), zp.clone()))
        return orig_final(zl, zp, *args, **kw)
    ddpm.sample_p_zs_given_zt, ddpm.sample_p_xh_given_z0 = step, last
    return calls, final


@pytest.mark.parametrize('resamplings', [1, 3])
def test_inpaint_reference_is_the_eager_iteration(resamplings):
    timesteps, n_lig = 4, [8, 6]
    ddpm = _oracle_ddpm(False, 8)
    tape = _Tape(ddpm, 11)
    calls, final = _record_reverse_calls(ddpm)
    lig, fixed = make_ligand(n_lig, 3)
    pocket = make_pocket()
    lig_n, poc_n = ddpm.normalize({k: v.clone() for k, v in lig.items()}, {k: v.clone() for k, v in pocket.items()})
    known = torch.cat([lig_n['x'], lig_n['one_hot']], 1)
    com0 = scatter_mean(poc_n['x'], poc_n['mask'])
    ddpm.inpaint(lig, pocket, fixed, resamplings=resamplings, timesteps=timesteps, center='ligand')
    sched = rc.conditional_schedule(timesteps, resamplings)
    assert len(calls) == len(sched)
    lm, pm = lig_n['mask'], poc_n['mask']
    draws = iter(tape.draws[1:])                                        # after the prior
    for k, r in enumerate(sched):
        n_rev, n1 = next(draws), next(draws)
        n2 = next(draws) if r.kind == 'inpaint_renoise' else None
        assert n_rev.shape == n1.shape == known.shape
        _, _, coef4 = rc.eager_coefficients(ddpm, False, r.s, timesteps, len(n_lig), 'cpu')
        (zu, pu) = calls[k][1]
        want_z, want_p = calls[k + 1][0] if k + 1 < len(calls) else final[0]
        got_z, got_p = rc.inpaint_update_ref(zu, pu, known, com0, fixed, n1, n2, coef4, lm, pm, torch.float32)
        assert torch.equal(got_z, want_z), f'replay {k} ({r.kind}, s={r.s}, u={r.u}): ligand'
        assert torch.equal(got_p, want_p), f'replay {k} ({r.kind}, s={r.s}, u={r.u}): pocket'


@pytest.mark.parametrize('resamplings,jump_length,timesteps', [(2, 2, 6), (3, 1, 4), (2, 3, 8)])
def test_joint_inpaint_reference_is_the_eager_iteration(resamplings, jump_length, timesteps):
    n_lig = [7, 5]
    ddpm = _oracle_ddpm(True, timesteps)
    tape = _Tape(ddpm, 12)
    calls, final = _record_reverse_calls(ddpm)
    lig, fixed = make_ligand(n_lig, 2)
    pocket = make_pocket()
    pfix = torch.ones(len(pocket['mask']))
    pfix[::3] = 0
    lig_n, poc_n = ddpm.normalize({k: v.clone() for k, v in lig.items()}, {k: v.clone() for k, v in pocket.items()})
    lm, pm = lig_n['mask'], poc_n['mask']
    mean_known = ddpm._fixed_com(lig_n['x'], poc_n['x'], fixed.bool(), pfix.bool(), lm, pm)
    x0l = torch.cat([lig_n['x'] - mean_known[lm], lig_n['one_hot']], 1)
    x0p = torch.cat([poc_n['x'] - mean_known[pm], poc_n['one_hot']], 1)
    ddpm.inpaint(lig, pocket, fixed, pfix, resamplings=resamplings, jump_length=jump_length)
    sched = rc.joint_schedule(resamplings, jump_length, timesteps)
    assert len(calls) == len(sched) and any(r.kind == 'inpaint_jump' for r in sched)
    draws = iter(tape.draws[3:])                                        # after the prior's three draws
    triple = lambda: tuple(next(draws) for _ in range(3))
    for k, r in enumerate(sched):
        n1, _ = triple(), triple()                                      # known part, reverse step
        n3 = triple() if r.kind == 'inpaint_jump' or r.eager_jump else None     # the eager loop jumps inside the step
        _, _, coef4 = rc.eager_coefficients(ddpm, True, r.s, timesteps, len(n_lig), 'cpu', jump_length)
        (zu, pu) = calls[k][1]
        want_l, want_p = calls[k + 1][0] if k + 1 < len(calls) else final[0]
        got_l, got_p = rc.joint_inpaint_update_ref(zu, pu, x0l, x0p, fixed, pfix, n1, n3, coef4, lm, pm, torch.float32)
        assert torch.equal(got_l, want_l), f'replay {k} ({r.kind}, s={r.s}, u={r.u}): ligand'
        assert torch.equal(got_p, want_p), f'replay {k} ({r.kind}, s={r.s}, u={r.u}): pocket'


def _eager_draw_ids(ddpm, fn):
    """Draw ids the eager loop sets, in order, while ``fn`` runs."""
    ids = []
    ddpm.loop_engine = 'eager'
    ddpm._draw_at = lambda stage, s=0, u=0, purpose=0: ids.append(seeded.draw_id(stage, s, u, purpose))
    fn()
    return ids


def _run_eager(name_or_spec):
    """The eager loop of a run of repaint_cases.RUNS (or a joint spec) on a small CPU batch with a zero denoiser."""
    spec = rc.RUNS[name_or_spec] if isinstance(name_or_spec, str) else name_or_spec
    joint = spec['joint']
    ddpm = _ddpm(joint, T, _ZeroDynamics(joint))
    lig, fixed = make_ligand([6, 4], 2)
    pocket = make_pocket()
    if name_or_spec == 'diversify':
        return _eager_draw_ids(ddpm, lambda: ddpm.diversify(lig, pocket, spec['noising_steps']))
    if joint:
        pfix = torch.ones(len(pocket['mask']))
        pfix[::3] = 0
        return _eager_draw_ids(ddpm, lambda: ddpm.inpaint(
            lig, pocket, fixed, pfix, resamplings=spec['resamplings'], jump_length=spec['jump_length'],
            return_frames=spec['frames'], timesteps=spec['timesteps']))
    return _eager_draw_ids(ddpm, lambda: ddpm.inpaint(lig, pocket, fixed, resamplings=spec['resamplings'],
                                                      timesteps=spec['timesteps'], center='ligand'))


@pytest.mark.parametrize('name', sorted(rc.RUNS))
def test_schedule_matches_eager_draws(name):
    first = seeded.STAGE_PARTIAL if name == 'diversify' else seeded.STAGE_PRIOR
    want = rc.draw_ids(rc.schedule_of(name), first)
    assert _run_eager(name) == want
    assert len(set(want)) == len(want), f'{name}: a draw id repeats'
    seq = rc.draw_sequence(name)
    assert len(set(seq)) == len(seq)
    if name == 'joint_frames':
        assert sum(r.eager_jump for r in rc.schedule_of(name)) == 5


# (resamplings, jump_length, timesteps): jump_length dividing T or not, a final partial block, one block only
REPAINT_EDGES = [(2, 10, 500), (3, 7, 500), (2, 3, 10), (2, 3, 11), (4, 5, 12), (3, 1, 4), (1, 1, 5), (3, 6, 6),
                 (3, 7, 6), (2, 4, 9)]


@pytest.mark.parametrize('resamplings,jump_length,timesteps', REPAINT_EDGES)
def test_joint_schedule_at_repaint_edges(resamplings, jump_length, timesteps):
    blocks = EnVariationalDiffusion.get_repaint_schedule(resamplings, jump_length, timesteps)
    sched = rc.joint_schedule(resamplings, jump_length, timesteps)
    # every jump back re-runs jump_length steps; the run starts at timesteps-1, ends at s = 0 and never leaves [0, T)
    assert len(sched) == sum(blocks) == timesteps + jump_length * (len(blocks) - 1)
    assert sched[0].s == timesteps - 1 and sched[-1].s == 0 and sched[-1].kind == 'inpaint'
    assert all(0 <= r.s < timesteps for r in sched)
    # a jump lands at most on timesteps-1: the t_back clamp of _joint_tables is never reached by a jump
    jumps = [r for r in sched if r.kind == 'inpaint_jump' or r.eager_jump]
    assert len(jumps) == len(blocks) - 1 and all(r.s + jump_length <= timesteps - 1 for r in jumps)
    assert [r.u for r in sched] == sorted(r.u for r in sched)
    spec = dict(resamplings=resamplings, jump_length=jump_length, timesteps=timesteps)
    ids = rc.draw_ids(sched)
    assert len(set(ids)) == len(ids)
    if timesteps < 100:
        assert _run_eager_sub(spec) == ids


def _run_eager_sub(spec):
    ddpm = _ddpm(True, spec['timesteps'], _ZeroDynamics(True))
    lig, fixed = make_ligand([6, 4], 2)
    pocket = make_pocket()
    pfix = torch.ones(len(pocket['mask']))
    return _eager_draw_ids(ddpm, lambda: ddpm.inpaint(lig, pocket, fixed, pfix, resamplings=spec['resamplings'],
                                                      jump_length=spec['jump_length']))


@pytest.mark.parametrize('timesteps,resamplings', [(50, 20), (500, 1), (3, 4), (1, 2)])
def test_conditional_schedule_has_no_repeated_draws(timesteps, resamplings):
    sched = rc.conditional_schedule(timesteps, resamplings)
    assert len(sched) == timesteps * resamplings
    assert [r.kind for r in sched].count('inpaint_last') == timesteps
    ids = rc.draw_ids(sched)
    assert len(set(ids)) == len(ids)


@pytest.mark.parametrize('timesteps', [50, 500])
def test_conditional_tables_match_eager_coefficients(timesteps):
    """Every row of _schedule_tables against the eager step's ops for that s; sub-sampled, t = (s+1)/timesteps looks the
    schedule up at round(t T) = (s+1) T / timesteps."""
    ddpm = _ddpm(False, T, _ZeroDynamics(False))
    t_table, coef = ddpm._schedule_tables(timesteps, timesteps, 'cpu')
    for s in range(timesteps):
        t, c3, c4 = rc.eager_coefficients(ddpm, False, s, timesteps, 1, 'cpu')
        assert int(torch.round(t_table[s] * T)) == (s + 1) * T // timesteps
        # one row here against a table computed on all rows at once: CPU vector and scalar paths round differently
        # (up to ~1e-5 after the expm1 cancellation); an off-by-one row or t_back moves a coefficient by more than 1e-3
        torch.testing.assert_close(coef[s], torch.cat((c3, c4), 1)[0], rtol=1e-4, atol=0)
        torch.testing.assert_close(t_table[s], t[0], rtol=3e-7, atol=0)


@pytest.mark.parametrize('jump_length,timesteps', [(10, 500), (7, 500), (1, 25), (3, 10)])
def test_joint_tables_clamp_t_back(jump_length, timesteps):
    """The RePaint columns of _joint_tables use t_back = min(s + jump_length, timesteps) at every row, clamped rows
    included."""
    ddpm = _ddpm(True, T, _ZeroDynamics(True))
    _, coef = ddpm._joint_tables(timesteps, jump_length, 'cpu')
    for s in range(timesteps):
        _, c3, c4 = rc.eager_coefficients(ddpm, True, s, timesteps, 1, 'cpu', jump_length)
        torch.testing.assert_close(coef[s], torch.cat((c3, c4), 1)[0], rtol=1e-4, atol=0, msg=f's={s}')
