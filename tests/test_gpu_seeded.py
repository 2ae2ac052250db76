"""GPU: seeded per-sample sampling.  The generator against its numpy restatement and in distribution; the denoiser's
batch invariance in deterministic mode in every math mode; regeneration of single ligands, bit for bit, alone and in other
batches, from every sampler and both loop engines; simulated GPU counts; the global generators left untouched."""
from argparse import Namespace

import numpy as np
import pytest
import torch

import seeded_cases as sc
from ddpm_cases import DDPM_CFG, HIST, JOINT_CFG, make_ligand, make_pocket
from stress_cases import LADDER_BIG, case_inputs, single_graph_inputs
from diffsbdd_b200 import _native, seeded, synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM
from diffsbdd_b200.config import FULLATOM_COND
from diffsbdd_b200.distributed import shard_bounds, shard_pocket, shard_seeds
from diffsbdd_b200.dynamics import EGNNDynamics
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion
from diffsbdd_b200.lightning_modules import LigandPocketDDPM

pytestmark = pytest.mark.gpu
FULL_LIG, FULL_POC = [25] * 64, [175] * 64          # configs[2]


# ---- 1. generator -----------------------------------------------------------------------------------------------------
LIG = np.repeat([0, 1, 2, 3], [3, 9, 1, 6])
POC = np.repeat([0, 1, 2, 3], [5, 2, 8, 4])
SEEDS = [0, 2 ** 63 - 1, 123456789012345, 42]


def _gpu(role, cols, kind, draw, seeds=SEEDS, lig=LIG, poc=POC):
    rows = {0: len(lig), 1: len(poc), 2: len(lig) + len(poc), 3: len(seeds)}[role]
    out = torch.empty((rows, cols), device='cuda')
    t = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.int64, device='cuda')
    seeded.fill(out, role, t(seeds), t([draw]), t(lig), t(poc), kind)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('role', [0, 1, 2, 3])
@pytest.mark.parametrize('cols', [1, 3, 4, 13])
def test_words_match_restatement(role, cols):
    draw = seeded.draw_id(seeded.STAGE_LOOP, 317, 5, seeded.PURPOSE_KNOWN) | (0x7 << 40)
    want = sc.words(role, cols, SEEDS, draw, LIG, POC)[:, :cols]
    got = _gpu(role, cols, _native.RNG_BITS, draw).cpu().view(torch.int32).numpy().view(np.uint32)
    assert np.array_equal(got, want)
    u = _gpu(role, cols, _native.RNG_UNIFORM, draw).cpu().numpy()
    assert np.array_equal(u, sc.uniform(want))
    z = _gpu(role, cols, _native.RNG_NORMAL, draw).cpu().numpy().astype(np.float64)
    zw = sc.normals(sc.words(role, cols, SEEDS, draw, LIG, POC))[:, :cols]
    # fp32 logf / sqrtf / sincospif against float64: within 8 ulp of max(|z|, 1)
    assert np.all(np.abs(z - zw) <= 8 * 2.0 ** -23 * np.maximum(np.abs(zw), 1.0)), float(np.abs(z - zw).max())


def test_normal_distribution_1e7():
    from scipy import stats
    n = 10_000_000
    z = _gpu(0, 8, _native.RNG_NORMAL, 99, seeds=[31337], lig=np.zeros(n // 8, int), poc=np.zeros(0, int)).cpu().numpy()
    z = z.astype(np.float64).ravel()
    assert abs(z.mean()) < 5 / np.sqrt(n)
    assert abs(z.var() - 1) < 5 * np.sqrt(2 / n)
    p_tail = 2 * stats.norm.sf(4)
    k = int((np.abs(z) > 4).sum())
    assert abs(k - n * p_tail) < 5 * np.sqrt(n * p_tail), (k, n * p_tail)
    assert stats.kstest(z, 'norm').pvalue > 1e-4


def test_graph_draws_independent_of_batch_position():
    draw = seeded.draw_id(seeded.STAGE_LOOP, 10, 0, 0)
    full = _gpu(2, 3, _native.RNG_NORMAL, draw)
    # graph 1 alone, and as the last graph of another batch
    alone = _gpu(2, 3, _native.RNG_NORMAL, draw, seeds=[SEEDS[1]], lig=np.zeros(9, int), poc=np.zeros(2, int))
    other = _gpu(2, 3, _native.RNG_NORMAL, draw, seeds=[5, SEEDS[1]], lig=np.repeat([0, 1], [4, 9]),
                 poc=np.repeat([0, 1], [7, 2]))
    nl = len(LIG)
    rows_full = torch.tensor(list(range(3, 12)) + [nl + 5, nl + 6])
    rows_other = torch.tensor(list(range(4, 13)) + [13 + 7, 13 + 8])
    assert torch.equal(full[rows_full], alone)
    assert torch.equal(full[rows_full], other[rows_other])


def test_capture_reads_draw_id_at_replay():
    out = torch.empty((len(LIG), 5), device='cuda')
    seeds = torch.tensor(SEEDS, device='cuda')
    d = torch.zeros(1, dtype=torch.int64, device='cuda')
    m = torch.tensor(LIG, device='cuda')
    seeded.fill(out, 0, seeds, d, m, None)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        seeded.fill(out, 0, seeds, d, m, None)
    res = []
    for v in (3, 8):
        d.fill_(v)
        g.replay()
        res.append(out.clone())
    assert torch.equal(res[0], _gpu(0, 5, 0, 3)) and torch.equal(res[1], _gpu(0, 5, 0, 8))


# ---- 2. denoiser batch invariance (deterministic mode) ----------------------------------------------------------------
def _net(cfg, sd, mode, det=True):
    net = EGNNDynamics.from_config(cfg, device='cuda')
    net.load_state_dict(sd)
    net.eval()
    net.math_mode = mode
    net.deterministic = det
    return net


def _call(net, inp):
    with torch.no_grad():
        a, r = net(*[x.cuda() for x in inp])
    torch.cuda.synchronize()
    return a.clone(), r.clone()


@pytest.mark.parametrize('mode', ['fp32', '3xtf32', '3xfp16'])
@pytest.mark.parametrize('name', ['ladder_h128', 'ladder_h256', 'configs2'])
def test_denoiser_alone_vs_batched_bitwise(name, mode):
    if name == 'configs2':
        cfg = FULLATOM_COND
        sd, inp, g = syn.synthetic_state_dict(cfg, 0), syn.synthetic_denoiser_inputs(cfg, FULL_LIG, FULL_POC, seed=1), 37
    else:
        (cfg, sd, inp), g = case_inputs(name), LADDER_BIG
    net = _net(cfg, sd, mode)
    out = _call(net, inp)
    one = _call(net, single_graph_inputs(inp, g))
    lm, pm = inp[3].cuda() == g, inp[4].cuda() == g
    assert torch.equal(one[0], out[0][lm]), f'{name} {mode} ligand: {float((one[0] - out[0][lm]).abs().max()):.3e}'
    assert torch.equal(one[1], out[1][pm]), f'{name} {mode} pocket'


@pytest.mark.parametrize('mode', [15, 7, 0])
def test_no_layout_dependent_launch(mode):
    """The per-launch comparison of the ladder graph alone vs batched (stop-after hook): no operation may differ."""
    import launch_cases as lc
    from test_gpu_launches import WRITES, regions_of, run_stopped
    cfg, sd, inp = case_inputs('ladder_h256')
    g = LADDER_BIG
    runs = {'batch': inp, 'alone': single_graph_inputs(inp, g)}
    rows = {'batch': torch.cat([inp[3] == g, inp[4] == g]).cuda(), 'alone': None}
    n_lig = int((inp[3] == g).sum())
    nets = {k: _net(cfg, sd, mode) for k in runs}
    xs = {k: [t.cuda() for t in v] for k, v in runs.items()}
    ops = lc.op_sequence(cfg, True)
    H = cfg.hidden_nf
    nrecv, nq = lc.nm_of(cfg) * H, 2 * lc.nm_of(cfg) * H
    for key in runs:
        run_stopped(nets[key], xs[key], -1)
    found = []
    for k in range(1, len(ops) + 1):
        op = ops[k - 1]
        if op.kind not in WRITES:
            continue
        st = {}
        for key in runs:
            run_stopped(nets[key], xs[key], k)
            dm, _, reg = regions_of(nets[key], xs[key], True)
            S = lc.read_state(nets[key]._workspace, reg, cfg, dm)
            sel = {}
            for n in WRITES[op.kind]:
                v = S[n] if rows[key] is None else S[n][rows[key]]
                if n == 'P' and op.kind == 'g1':
                    v = v[:, nq:nq + 2 * H]
                if n == 'P' and op.kind == 'g4':
                    ncol = nq + (2 * H if op.layer + 1 < cfg.n_layers else 0)
                    v = torch.cat([v[:, nrecv:ncol].flatten(), v[:n_lig, :nrecv].flatten()])
                sel[n] = v.contiguous().view(torch.int32).clone()
            st[key] = sel
        diff = [n for n in st['batch'] if not torch.equal(st['batch'][n], st['alone'][n])]
        if diff:
            found.append((k - 1, op.kind, op.layer, op.sub, diff))
    assert not found, found


# ---- 3. regeneration ------------------------------------------------------------------------------------------------------
def _ddpm(cfg, T, mode='fp32', joint=False, engine='graph', seed=0):
    dyn = _net(cfg, syn.synthetic_state_dict(cfg, seed), mode)
    cls = EnVariationalDiffusion if joint else ConditionalDDPM
    ddpm = cls(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=T,
               noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2', norm_values=(1, 4), size_histogram=HIST)
    ddpm.loop_engine = engine
    return ddpm.cuda().eval()


def _pick(d, idx):
    """Sub-batch of a ligand/pocket dict with the graphs idx (in that order), renumbered from 0."""
    parts = [shard_pocket(d, i, i + 1) for i in idx]
    out = {k: torch.cat([p[k] for p in parts]) for k in ('x', 'one_hot', 'size')}
    out['mask'] = torch.cat([p['mask'] + j for j, p in enumerate(parts)])
    return out


def _copy(d):
    return {k: v.clone() for k, v in d.items()}


def _rows(out, mask, g, frames):
    return out[:, mask == g] if frames > 1 else out[mask == g]


def _check_regen(run, n, picks, frames=1, pocket_too=True):
    """run(idx) -> sampler outputs for the graphs idx; graph idx[k] of every pick must equal the full batch bit for bit."""
    full = run(list(range(n)))
    for idx in picks:
        sub = run(idx)
        for k, g in enumerate(idx):
            assert torch.equal(_rows(sub[0], sub[2], k, frames), _rows(full[0], full[2], g, frames)), (idx, g, 'ligand')
            if pocket_too:
                assert torch.equal(_rows(sub[1], sub[3], k, frames), _rows(full[1], full[3], g, frames)), (idx, g, 'pocket')
    return full


def test_regenerate_configs2_500_steps_3xfp16():
    cfg = FULLATOM_COND
    ddpm = _ddpm(cfg, 500, '3xfp16')
    data = syn.synthetic_complex_batch(cfg, FULL_LIG, FULL_POC, seed=3)
    pocket = {'x': data['pocket_coords'].cuda(), 'one_hot': data['pocket_one_hot'].cuda(),
              'size': data['num_pocket_nodes'].cuda(), 'mask': data['pocket_mask'].cuda()}
    n_lig = torch.tensor(FULL_LIG).cuda()
    seeds = torch.arange(1000, 1064)
    run = lambda idx: ddpm.sample_given_pocket(_pick(_copy(pocket), idx), n_lig[idx], return_frames=5, seeds=seeds[idx])
    full = _check_regen(run, 64, [[0], [37], [63], [63, 37, 12, 5, 0]], frames=5)
    assert torch.isfinite(full[0]).all()


@pytest.mark.parametrize('engine', ['graph', 'eager'])
@pytest.mark.parametrize('mode', ['fp32', '3xtf32', '3xfp16'])
def test_regenerate_sample_small(mode, engine):
    cfg = FULLATOM_COND.with_(n_layers=2)
    ddpm = _ddpm(cfg, 12, mode, engine=engine)
    pocket = syn.synthetic_pocket(cfg, [30, 22, 41, 17, 26], seed=5, spread=3.0)
    pocket = {k: v.cuda() for k, v in pocket.items()}
    n_lig = torch.tensor([7, 5, 9, 4, 6]).cuda()
    seeds = torch.tensor([11, 2 ** 62, 3, 4, 5])
    run = lambda idx: ddpm.sample_given_pocket(_pick(_copy(pocket), idx), n_lig[idx], return_frames=3, seeds=seeds[idx])
    _check_regen(run, 5, [[2], [4, 2, 0]], frames=3)
    run1 = lambda idx: ddpm.sample_given_pocket(_pick(_copy(pocket), idx), n_lig[idx], seeds=seeds[idx])
    _check_regen(run1, 5, [[3], [3, 1]])




@pytest.mark.parametrize('engine', ['graph', 'eager'])
def test_regenerate_inpaint_and_diversify(engine):
    ddpm = _ddpm(DDPM_CFG, 10, engine=engine, seed=5)
    pocket = make_pocket('cuda')
    lig, fixed = make_ligand([8, 6], 3, device='cuda')
    seeds = torch.tensor([77, 78])

    def inp(idx):
        sel = torch.cat([fixed[lig['mask'] == i] for i in idx])
        return ddpm.inpaint(_pick(_copy(lig), idx), _pick(_copy(pocket), idx), sel, resamplings=3, seeds=seeds[idx])

    def div(idx):
        return ddpm.diversify(_pick(_copy(lig), idx), _pick(_copy(pocket), idx), noising_steps=4, seeds=seeds[idx])
    _check_regen(inp, 2, [[1], [1, 0]])
    _check_regen(div, 2, [[0], [1, 0]])


@pytest.mark.parametrize('engine', ['graph', 'eager'])
def test_regenerate_joint(engine):
    ddpm = _ddpm(JOINT_CFG, 8, joint=True, engine=engine, seed=6)
    n_lig, n_poc = torch.tensor([6, 4, 5]).cuda(), torch.tensor([14, 11, 9]).cuda()
    seeds = torch.tensor([5, 6, 7])
    run = lambda idx: ddpm.sample(len(idx), n_lig[idx], n_poc[idx], device='cuda', seeds=seeds[idx])
    _check_regen(run, 3, [[1], [2, 0]])
    lig, lfix = make_ligand([7, 5], 2, device='cuda')
    pocket = make_pocket('cuda')
    pfix = torch.ones(len(pocket['mask']), device='cuda')
    pfix[::3] = 0

    def inp(idx):
        lf = torch.cat([lfix[lig['mask'] == i] for i in idx])
        pf = torch.cat([pfix[pocket['mask'] == i] for i in idx])
        return ddpm.inpaint(_pick(_copy(lig), idx), _pick(_copy(pocket), idx), lf, pf, resamplings=2, jump_length=2,
                            seeds=seeds[:2][idx])
    _check_regen(inp, 2, [[1], [1, 0]])


def test_regenerate_generate_ligand_tensors_with_size_prior():
    cfg = FULLATOM_COND.with_(n_layers=2)
    egnn = Namespace(device='cuda', **{k: v for k, v in cfg.kwargs().items()
                                       if k not in ('atom_nf', 'residue_nf', 'n_dims', 'condition_time', 'mode',
                                                    'update_pocket_coords')})
    diff = Namespace(diffusion_steps=16, diffusion_noise_schedule='polynomial_2', diffusion_noise_precision=5.0e-4,
                     diffusion_loss_type='l2', normalize_factors=[1, 4])
    hist = np.random.default_rng(0).random((27, 177)).tolist()
    model = LigandPocketDDPM(outdir=None, dataset='crossdock', datadir=None, batch_size=4, lr=1e-3, egnn_params=egnn,
                             diffusion_params=diff, num_workers=0, augment_noise=0, augment_rotation=False, clip_grad=True,
                             eval_epochs=1, eval_params=Namespace(), visualize_sample_epoch=1, visualize_chain_epoch=1,
                             auxiliary_loss=False, loss_params=Namespace(), mode='pocket_conditioning',
                             node_histogram=hist, pocket_representation='full-atom')
    model.ddpm.dynamics.load_state_dict(syn.synthetic_state_dict(cfg, 0))
    model = model.to('cuda').eval()
    model.ddpm.dynamics.deterministic = True
    pocket = {k: v.cuda() for k, v in syn.synthetic_pocket(cfg, [30, 22, 41, 17], seed=5, spread=3.0).items()}
    seeds = torch.tensor([9, 8, 7, 6])
    run = lambda idx: model.generate_ligand_tensors(_pick(_copy(pocket), idx), n_nodes_min=2, seeds=seeds[idx])
    full = _check_regen(run, 4, [[2], [3, 0, 2]])
    # the sizes are the restated inverse-CDF draws of the seeded uniforms
    u = _gpu(3, 1, _native.RNG_UNIFORM, seeded.draw_id(seeded.STAGE_SIZE), seeds=seeds.tolist(), lig=np.zeros(0, int),
             poc=np.zeros(0, int)).cpu().numpy().ravel()
    prob = model.ddpm.size_distribution.prob.numpy()
    want = np.maximum(sc.expected_sizes(prob, [30, 22, 41, 17], u), 2)
    assert torch.bincount(full[2]).tolist() == want.tolist()


# ---- 4. GPU count, duplicates, global generators -------------------------------------------------------------------------
def test_world_sizes_give_identical_ligands():
    cfg = FULLATOM_COND.with_(n_layers=2)
    ddpm = _ddpm(cfg, 10, '3xfp16')
    n = 8
    pocket = {k: v.cuda() for k, v in syn.synthetic_pocket(cfg, [20 + 3 * i for i in range(n)], seed=8, spread=3.0).items()}
    n_lig = torch.tensor([4 + i % 4 for i in range(n)]).cuda()
    seeds = torch.arange(500, 500 + n)
    gathered = {}
    for world in (1, 2, 3, 8):
        parts = []
        for r in range(world):
            lo, hi = shard_bounds(n, world, r)
            if hi > lo:
                parts.append(ddpm.sample_given_pocket(shard_pocket(_copy(pocket), lo, hi), n_lig[lo:hi],
                                                      seeds=shard_seeds(seeds, lo, hi))[0])
        gathered[world] = torch.cat(parts)
    for w in (2, 3, 8):
        assert torch.equal(gathered[w], gathered[1]), w


def test_same_seed_same_ligand_and_rng_untouched():
    cfg = FULLATOM_COND.with_(n_layers=2)
    ddpm = _ddpm(cfg, 10, '3xfp16')
    one = syn.synthetic_pocket(cfg, [25], seed=9, spread=3.0)
    pocket = {k: torch.cat([v, v + (1 if k == 'mask' else 0)]).cuda() if k != 'size' else torch.cat([v, v]).cuda()
              for k, v in one.items()}
    cpu_state, gpu_state = torch.get_rng_state(), torch.cuda.get_rng_state()
    for engine in ('graph', 'eager'):
        ddpm.loop_engine = engine
        out = ddpm.sample_given_pocket(_copy(pocket), torch.tensor([6, 6]).cuda(), seeds=[4242, 4242])
        assert torch.equal(out[0][out[2] == 0], out[0][out[2] == 1]), engine
    assert torch.equal(torch.get_rng_state(), cpu_state)
    assert torch.equal(torch.cuda.get_rng_state(), gpu_state)
    # an unseeded call still draws from the global generator
    ddpm.sample_given_pocket(_copy(pocket), torch.tensor([6, 6]).cuda())
    assert not torch.equal(torch.cuda.get_rng_state(), gpu_state)


def _twice(fn, what):
    """The first call captures the step graphs, the second replays the cached ones: both must give the same bits."""
    a = fn()
    b = fn()
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), f'{what}: output {i} differs between the capturing and the replaying call'


def test_capturing_and_replaying_calls_agree():
    ddpm = _ddpm(DDPM_CFG, 10, seed=5)
    pocket = make_pocket('cuda')
    lig, fixed = make_ligand([8, 6], 3, device='cuda')
    seeds = torch.tensor([77, 78])
    _twice(lambda: ddpm.inpaint(_copy(lig), _copy(pocket), fixed, resamplings=3, seeds=seeds), 'inpaint r3')
    assert next(iter(ddpm._graph_cache.values()))['seeded']
    _twice(lambda: ddpm.diversify(_copy(lig), _copy(pocket), noising_steps=4, seeds=seeds), 'diversify')
    _twice(lambda: ddpm.sample_given_pocket(_copy(pocket), torch.tensor([7, 5]).cuda(), return_frames=2, seeds=seeds),
           'sample_given_pocket')
    joint = _ddpm(JOINT_CFG, 8, joint=True, seed=6)
    lig, lfix = make_ligand([7, 5], 2, device='cuda')
    pfix = torch.ones(len(pocket['mask']), device='cuda')
    pfix[::3] = 0
    _twice(lambda: joint.inpaint(_copy(lig), _copy(pocket), lfix, pfix, resamplings=2, jump_length=2, seeds=seeds),
           'joint inpaint r2 j2')
    _twice(lambda: joint.inpaint(_copy(lig), _copy(pocket), lfix, pfix, resamplings=3, jump_length=1, seeds=seeds),
           'joint inpaint r3 j1')
    _twice(lambda: joint.sample(2, torch.tensor([6, 4]).cuda(), torch.tensor([14, 11]).cuda(), device='cuda', seeds=seeds),
           'joint sample')
