"""GPU: the single-product FP16 math mode ('1xfp16', mask 31): x.w ~= x_hi.w_hi on wgmma, held to float64 at its own
error bound (tests/fast_math_cases.py).

1. Per launch, against float64, on the eleven cases of test_gpu_launches.py, deterministic and default mode: every output
   within twice the worst-case bound of ``fast_math_cases.Arith1x``, and its RMS error at most R_TC times the RMS error of
   the float64 evaluation on operands rounded to fp16 as the kernel rounds them (launches without a tensor-core
   contraction: R_FP32 times a plain fp32 evaluation, the budget of math mode 0).
2. Whole forward: every golden of width 128, 192 or 256 and configs[2] against the float64 oracle; mode 31 must differ
   from mode 15 (the new kernels ran).
3. Deterministic mode: a call repeats bit for bit; a graph alone and inside its batch give the same bits.
4. Graph engine: a seeded 50-step ``sample_given_pocket``; every replay equals the eager denoiser plus the fused update
   bit for bit, and switching 15 -> 31 -> 15 re-captures and reproduces each mode's own output.
5. Sample level (configs[2], 500 steps): the distributions of mode 31 and mode 15 samples agree (two-sample KS tests,
   chi-square on atom types).
6. Errors: bit 16 without bit 8, H = 64 and sin_embedding are rejected; an activation beyond the fp16 range raises.

Measured on one H100 80GB HBM3 at a 700 W power limit:
* per launch, largest value over the cases, layers and both modes: the RMS ratio of every single-product launch (g1-g4,
  gcl, coord) to the rounded-operand evaluation is 1.00 (the kernel's error is the operand rounding; the fp32
  accumulation adds nothing visible), so R_TC = 1.3 keeps the margin of test_gpu_launches.py; the other launches reach
  3.57 (post) against plain fp32, as in mode 15.  Max error over twice the worst-case bound: 0.24 (g1, binade sweep) on
  the contractions, 0.50 on the single-rounding steps finish and post.
* planted defects, each built once and then reverted (deterministic per-launch test):
  - the last of the four k-steps of every chunk dropped in ``mma_chunk``: fails on all 8 cases, coord up to 5 800 x;
  - activations truncated instead of rounded to fp16 in ``store_pair``: fails on all 8 cases against R_TC = 1.3
    (largest ratio per case 2.0 (binade sweep, gcl) to 4.8 (emb8_h256_l3, coord)).
* the three cases added for width 192 and the edge-type table at 128 (moad, joint_fc_h192, tb_noatt_notanh_h128):
  every single-product launch 1.00 against the rounded-operand evaluation, max error over twice the bound 0.089 (g3,
  tb_noatt_notanh_h128) on the contractions; the other launches reach 2.48 (post) and 1.33 (finish, joint_fc_h192)
  against plain fp32.  Planted defects in their instances, each built once and then reverted:
  - H = 192: the last k-step of a tile's last chunk dropped in ``mma_chunk``: fails on moad and joint_fc_h192,
    deterministic and default mode, coord up to 10 989 x, every other contraction 303-1 627 x;
  - attention off: a gate of 1 - 2^-12 instead of 1: fails on tb_noatt_notanh_h128, both modes, gcl 1.57 x;
  - the edge-type table term scaled by 1 - 2^-10 at H = 128 passes here (gcl 1.06, coord 1.13): the change is below the
    fp16 rounding of the operand it is added into, which the single-product model accepts; modes 15 and 7 catch it
    (test_gpu_launches.py).
* whole forward against the float64 oracle, max |error| / max |output| per output block: at most 1.1e-3 (sub2_h256_l2
  and reflect_h256_l3 ligand velocity, outputs ~0.03); configs[2]: ligand velocity max 1.2e-4 (RMS 2.3e-5, outputs up
  to 0.24), ligand h max 1.2e-5 (RMS 2.0e-6), pocket h max 6.1e-6.  FWD_REL = 3e-3.
* 500-step configs[2] samples, 1,600 ligand atoms per run: KS distance mode 31 vs mode 15 on the same seeds 0.004 for
  both distance distributions, against 0.028 / 0.046 between two mode-15 runs on different seeds (critical value
  0.058); atom-type chi-square p = 1.0; per-ligand coordinate RMSD 31 vs 15 median 0.015 A (max 0.022 A), no atom type
  changed.
The file (51 tests) takes 28 s on that card.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from scipy import stats

import fast_math_cases as fm
import launch_cases as lc
from helpers import golden_cases, load_golden
from stress_cases import LADDER_BIG, case_inputs, single_graph_inputs
from test_gpu_launches import CASES, DEFAULT_MODE_CASES, READS_ONLY, SAFETY, Runner, case_cfg
from trajectory_cases import full_pocket, ligand_update, make_ddpm, record_conditional
from diffsbdd_b200 import _native, synthetic as syn
from diffsbdd_b200.config import FULLATOM_COND, DynamicsConfig
from diffsbdd_b200.dynamics import EGNNDynamics
from oracle import egnn_oracle

pytestmark = pytest.mark.gpu

MODE = fm.MODE
R_TC = 1.3         # single-product launches vs the float64 evaluation on fp16-rounded operands (measured 1.00)
R_FP32 = 8.0       # launches without a tensor-core contraction vs plain fp32 (the mode-0 budget of test_gpu_launches.py)
TC_KINDS = ('g1', 'g2', 'g3', 'g4', 'gcl', 'coord')
RESULTS = []


@pytest.fixture(autouse=True, scope='module')
def _no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old
    if RESULTS:
        print('\nper-launch results (mode 31): case det kind  max RMS ratio  max err/bound')
        agg = {}
        for case, det, kind, rr, br in RESULTS:
            a = agg.get((case, det, kind), (0.0, 0.0))
            agg[(case, det, kind)] = (max(a[0], rr), max(a[1], br))
        for k, (rr, br) in sorted(agg.items()):
            print(f'  {k[0]:34s} {int(k[1])} {k[2]:8s} {rr:7.2f} {br:7.3f}')


def make_net(cfg, sd, mode=MODE, det=True):
    net = EGNNDynamics.from_config(cfg, device='cuda')
    net.load_state_dict(sd)
    net.eval()
    net.math_mode = mode
    net.deterministic = det
    return net


def call(net, inp):
    with torch.no_grad():
        a, r = net(*[x.cuda() for x in inp])
    torch.cuda.synchronize()
    return a.clone(), r.clone()


# ---- 1. per launch --------------------------------------------------------------------------------------------------
class Runner1x(Runner):
    """test_gpu_launches.Runner in mode 31: the single-product model in the float64 restatement, and the rounded-operand
    evaluation as the statistical reference."""

    def __init__(self, name, det):
        super().__init__(name, MODE, det)
        fm.single_product(self.r64)
        self.r32 = fm.RoundedRestater(self.cfg, self.sd, self.inp, MODE, 'cuda')

    def check_unit(self, op, Sb, Sa):
        o64, oref = self.r64.run(op, Sb), self.r32.run(op, Sb)
        budget = R_TC if op.kind in TC_KINDS else R_FP32
        for name, entry in o64.items():
            v64, b64 = entry[0], entry[1]
            if name in ('out_atoms', 'out_residues'):
                got = self.full[0] if name == 'out_atoms' else self.full[1]
            else:
                got = lc.output_view(Sa, name, entry)
            got = got.double()
            what = f'{self.name} mode 31 det {int(self.det)} {op.kind} l{op.layer} s{op.sub} {name}'
            if b64 is None:
                assert torch.equal(got, v64.to(got.dtype)), what
                continue
            live = torch.ones_like(got, dtype=torch.bool)
            if op.kind == 'g4' and name == 'P':
                live = ~lc.dead_p_mask(self.cfg, self.dm, MODE, got.shape[1]).cuda()
            err = (got - v64).abs()[live]
            assert torch.isfinite(err).all(), what
            if not err.numel():
                continue
            br = float((err / (SAFETY * b64[live] + 1e-300)).max())
            rms_k = float(err.pow(2).mean().sqrt())
            rms_ref = float((oref[name][0].double() - v64)[live].pow(2).mean().sqrt())
            rr = rms_k / rms_ref if rms_ref > 0 else (0.0 if rms_k == 0 else math.inf)
            RESULTS.append((self.name, self.det, op.kind, rr, br))
            if br > 1.0:
                self.failures.append(f'{what}: error {br:.2f} x the worst-case bound')
            if rr > budget:
                self.failures.append(f'{what}: RMS error {rms_k:.3e} = {rr:.2f} x the reference evaluation ({rms_ref:.3e})')


def _cases():
    return [name for name in CASES if lc.effective_mode(case_cfg(name), MODE) == MODE]


CASES_1X = _cases()
DEFAULT_CASES_1X = [n for n in CASES_1X if n in DEFAULT_MODE_CASES]


@pytest.mark.parametrize('name', CASES_1X)
def test_launches_deterministic(name):
    r = Runner1x(name, True)
    prev_stop, prev_ws = None, None
    for i, j, op in lc.launch_units(r.cfg, True):
        before = prev_ws if prev_stop == i else r.snapshot(i)
        after = r.snapshot(j)
        r.check_unit(op, r.state(before), r.state(after))
        prev_stop, prev_ws = j, after
    assert not r.failures, '\n'.join(r.failures)


@pytest.mark.parametrize('name', DEFAULT_CASES_1X)
def test_launches_default_mode(name):
    r = Runner1x(name, False)
    for i, j, op in lc.launch_units(r.cfg, False):
        if op.kind not in READS_ONLY:
            continue
        S = r.state(r.snapshot(j))
        r.check_unit(op, S, S)
    assert not r.failures, '\n'.join(r.failures)


# ---- 2. whole forward -----------------------------------------------------------------------------------------------
# max |error| against float64 relative to max |float64 output|, per output block (ligand / pocket x vel / h)
FWD_REL = 3e-3


def _fwd_errors(got, want):
    out = {}
    for side, g, w in (('lig', got[0], want[0]), ('poc', got[1], want[1])):
        for cols, sl in (('vel', slice(0, 3)), ('h', slice(3, None))):
            e = (g[:, sl].double().cpu() - w[:, sl].cpu()).abs()
            if e.numel():
                out[f'{side} {cols}'] = (float(e.max()), float(e.pow(2).mean().sqrt()), float(w[:, sl].abs().max()))
    return out


def _fwd_cases():
    out = [n for n in golden_cases() if lc.effective_mode(load_golden(n)[0], MODE) == MODE]
    return out + ['configs2']


@pytest.mark.parametrize('name', _fwd_cases())
def test_forward_against_float64(name):
    if name == 'configs2':
        cfg, sd, inp = lc.configs2_case()
    else:
        cfg, sd, inp = load_golden(name)[:3]
    net = make_net(cfg, sd, MODE, det=True)
    got = call(net, inp)
    assert net.math_mode == MODE
    want = egnn_oracle.denoiser_forward(cfg, sd, *inp, dtype=torch.float64, device='cuda')
    errs = _fwd_errors(got, want)
    print(f'\n{name}: ' + '  '.join(f'{k} max {m:.2e} rms {r:.2e} (|ref| {s:.2e})' for k, (m, r, s) in errs.items()))
    for k, (m, r, s) in errs.items():
        assert m <= FWD_REL * max(s, 1e-3), f'{name} {k}: max error {m:.3e} vs output scale {s:.3e}'
    net.math_mode = 15
    ref15 = call(net, inp)
    assert not torch.equal(got[0], ref15[0]), f'{name}: mode 31 gave the mode-15 output (the single-product path did not run)'


# ---- 3. deterministic mode ------------------------------------------------------------------------------------------
def test_repeat_bitwise():
    cfg, sd, inp = lc.configs2_case()
    net = make_net(cfg, sd)
    a, b = call(net, inp), call(net, inp)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize('name', ['ladder_h128', 'ladder_h256', 'configs2'])
def test_alone_vs_batched_bitwise(name):
    if name == 'configs2':
        cfg = FULLATOM_COND
        sd, inp, g = syn.synthetic_state_dict(cfg, 0), syn.synthetic_denoiser_inputs(cfg, [25] * 64, [175] * 64, seed=1), 37
    else:
        (cfg, sd, inp), g = case_inputs(name), LADDER_BIG
    net = make_net(cfg, sd)
    out = call(net, inp)
    one = call(net, single_graph_inputs(inp, g))
    lm, pm = inp[3].cuda() == g, inp[4].cuda() == g
    assert torch.equal(one[0], out[0][lm]), f'{name} ligand: {float((one[0] - out[0][lm]).abs().max()):.3e}'
    assert torch.equal(one[1], out[1][pm]), f'{name} pocket'


# ---- 4. graph engine ------------------------------------------------------------------------------------------------
def test_graph_replays_match_eager_denoiser_and_fused_update():
    ddpm = make_ddpm(FULLATOM_COND, False, timesteps=50)
    ddpm.dynamics.math_mode = '1xfp16'
    pocket, n_lig = full_pocket()
    rec = record_conditional(ddpm, pocket, n_lig, seed=77)
    dyn, lm, pm = ddpm.dynamics, rec['lig_mask'], rec['pocket_mask']
    assert dyn.math_mode == MODE and len(rec['step']) == 50
    for k, s in enumerate(rec['step']):
        with torch.no_grad():
            eps_l, _ = dyn(rec['z'][k], rec['pocket'][k], rec['t'][k], lm, pm)
        got = ligand_update(ddpm, rec['z'][k], eps_l, rec['noise'][k], rec['coef3'][k], rec['pocket'][k], lm, pm)
        assert torch.equal(got[0], rec['z'][k + 1]) and torch.equal(got[1], rec['pocket'][k + 1]), \
            f'step s={s}: eager denoiser + fused update differs from the graph replay'


def test_mode_switch_recaptures():
    ddpm = make_ddpm(FULLATOM_COND, False, timesteps=50)
    pocket, n_lig = full_pocket()

    def run(mode):
        ddpm.dynamics.math_mode = mode
        torch.manual_seed(5)
        out = ddpm.sample_given_pocket({k: v.clone() for k, v in pocket.items()}, n_lig)
        return out, next(iter(ddpm._graph_cache.values()))['graphs']['reverse']

    a15, g15 = run('3xfp16')
    a31, g31 = run('1xfp16')
    b15, g15b = run('3xfp16')
    assert g31 is not g15 and g15b is not g31
    assert not torch.equal(a31[0], a15[0])
    for x, y in zip(a15, b15):
        assert torch.equal(x, y), 'mode 15 after a mode-31 run does not reproduce its own output'
    b31, _ = run('1xfp16')
    for x, y in zip(a31, b31):
        assert torch.equal(x, y), 'mode 31 does not reproduce its own output'


# ---- 5. sample level ------------------------------------------------------------------------------------------------
def _sample(ddpm, pocket, n_lig, seeds, mode):
    ddpm.dynamics.math_mode = mode
    return ddpm.sample_given_pocket({k: v.clone() for k, v in pocket.items()}, n_lig, seeds=seeds)


def _features(out, atom_nf):
    """Per ligand atom: nearest other ligand atom distance, nearest pocket atom distance, atom type."""
    xh, mask = out[0], out[2]
    x, types = xh[:, :3].double(), xh[:, 3:3 + atom_nf].argmax(1)
    nn, npk = [], []
    for g in range(int(mask.max()) + 1):
        xl, xp = x[mask == g], out[1][out[3] == g][:, :3].double()
        d = torch.cdist(xl, xl)
        d.fill_diagonal_(float('inf'))
        nn.append(d.min(1).values)
        npk.append(torch.cdist(xl, xp).min(1).values)
    return torch.cat(nn).cpu().numpy(), torch.cat(npk).cpu().numpy(), types.cpu().numpy()


def test_sample_distributions_match_mode_15():
    """configs[2], deterministic, graph engine, 500 steps: mode 31 and mode 15 on the same 64 seeds, and mode 15 on 64
    other seeds for the scale of independent runs."""
    cfg = FULLATOM_COND
    ddpm = make_ddpm(cfg, False, timesteps=500)
    pocket, n_lig = full_pocket()
    seeds, other = torch.arange(5000, 5064), torch.arange(9000, 9064)
    runs = {'15': _sample(ddpm, pocket, n_lig, seeds, '3xfp16'), '31': _sample(ddpm, pocket, n_lig, seeds, '1xfp16'),
            '15b': _sample(ddpm, pocket, n_lig, other, '3xfp16')}
    feats = {k: _features(v, cfg.atom_nf) for k, v in runs.items()}
    n = len(feats['15'][0])
    crit = 1.628 * math.sqrt(2.0 / n)                       # two-sample KS, alpha = 0.01, n = m
    report = []
    for i, what in enumerate(('nearest ligand neighbour', 'nearest pocket atom')):
        d31 = stats.ks_2samp(feats['31'][i], feats['15'][i]).statistic
        dind = stats.ks_2samp(feats['15b'][i], feats['15'][i]).statistic
        report.append(f'{what}: KS 31 vs 15 {d31:.4f}, independent 15 vs 15 {dind:.4f} (critical {crit:.4f})')
        assert d31 < crit, report[-1]
    cnt = np.stack([np.bincount(feats[k][2], minlength=cfg.atom_nf) for k in ('31', '15')])
    cnt = cnt[:, cnt.sum(0) > 0]
    chi = stats.chi2_contingency(cnt)
    report.append(f'atom types: chi-square p = {chi.pvalue:.3f}')
    assert chi.pvalue > 0.01, report[-1]
    lm = runs['15'][2]
    rmsd = [float((runs['31'][0][lm == g, :3] - runs['15'][0][lm == g, :3]).pow(2).sum(1).mean().sqrt()) for g in range(64)]
    changed = float((feats['31'][2] != feats['15'][2]).mean())
    report.append(f'per-ligand coordinate RMSD 31 vs 15: median {np.median(rmsd):.3f}, max {max(rmsd):.3f}; '
                  f'atom types changed: {changed:.3f}')
    print('\n' + '\n'.join(report))


# ---- 6. errors ------------------------------------------------------------------------------------------------------
def _handle(cfg):
    net = EGNNDynamics.from_config(cfg, device='cuda')
    net.load_state_dict(syn.synthetic_state_dict(cfg, 0))
    net.eval()
    inp = syn.synthetic_denoiser_inputs(cfg, [5], [9], seed=0)
    net.math_mode = 0
    call(net, inp)
    return net


@pytest.mark.parametrize('mask', [16, 17, 32, -1])
def test_bad_masks_rejected(mask):
    net = _handle(DynamicsConfig(joint_nf=16, hidden_nf=128, n_layers=1))
    lib = _native.load()
    assert lib.dsb_dynamics_set_math_mode(C.c_void_p(net._handle), mask) == -1      # DSB_ERR_INVALID_ARGUMENT
    assert lib.dsb_dynamics_set_math_mode(C.c_void_p(net._handle), 31) == 0


@pytest.mark.parametrize('cfg', [DynamicsConfig(joint_nf=16, hidden_nf=64, n_layers=1),
                                 DynamicsConfig(joint_nf=16, hidden_nf=128, n_layers=1, sin_embedding=True)],
                         ids=['h64', 'sin_embedding'])
def test_unsupported_configs_rejected(cfg):
    net = _handle(cfg)
    with pytest.raises(Exception):
        net.math_mode = '1xfp16'
    assert _native.load().dsb_dynamics_set_math_mode(C.c_void_p(net._handle), 31) == -2     # DSB_ERR_UNSUPPORTED_CONFIG


def test_activation_beyond_fp16_range_raises():
    cfg, sd, inp = lc.configs2_case()
    sd = dict(sd)
    sd['egnn.embedding.weight'] = sd['egnn.embedding.weight'] * 1e5       # h beyond 65504 in the first node GEMM
    net = make_net(cfg, sd)
    with pytest.raises(ValueError, match='NaN detected in EGNN output'):
        with torch.no_grad():
            net(*[x.cuda() for x in inp])
        net.check_status()
