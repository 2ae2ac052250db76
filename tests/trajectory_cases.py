"""Recorded sampling trajectories of the production graph engine, and planted cut-off boundary pairs.

Recorder.  ``record_conditional`` / ``record_joint`` run an ordinary ``sample_given_pocket`` / ``sample`` call in which the
reverse loop (``ConditionalDDPM._graphed_reverse_steps`` / ``EnVariationalDiffusion._graphed_joint_reverse_steps``) is
replaced, for the duration of the call, by a copy that drives the same engine (``_engine`` / ``_joint_engine``), the same
captured graph (``_graph`` / ``_joint_graph``) and one ``g.replay()`` per step, and copies the static buffers around every
replay.  The prior, the normalisation and the final t = 0 step (``sample_p_xh_given_z0``) run unchanged.  In
deterministic mode the recorded run and an unmodified call with the same seed give the same bits, which shows that the
recorder ran the production path.

Each record holds, for the k-th replay (s = T-1-k): the state before it (``z[k]``, ``pocket[k]``; ``z[T]``, ``pocket[T]``
is the input of the t = 0 call), the step counter ``step[k]`` read before the replay, and what the replay wrote into its
static buffers: ``t[k]``, ``coef3[k]`` and the noise it drew (``noise[k]``: ``st['noise']``, or the joint ``st['n_rev']``
triple).

Planted pairs.  ``planted_batch`` places, for each block type (ligand-ligand, pocket-pocket, ligand-pocket), one pair per
graph at a stated float64 distance from that block's cut-off: exactly at the cut-off, at nextafter(cut, +-inf) and at
cut +- {2, 4, 16, 256} ulp, along a coordinate axis and along generic directions 10-30 A from the origin.
"""
import ctypes as C
import math

import numpy as np
import torch

from ddpm_cases import HIST
from diffsbdd_b200 import _native, synthetic as syn
from diffsbdd_b200.conditional_model import ConditionalDDPM
from diffsbdd_b200.config import FULLATOM_COND, DynamicsConfig
from diffsbdd_b200.dynamics import EGNNDynamics
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion, scatter_mean

T = 500
COND_LIG, COND_POC = [25] * 64, [175] * 64       # configs[2]: 64 complexes of 25 + 175 atoms
JOINT_LIG, JOINT_POC = [25] * 16, [175] * 16     # joint model: 16 graphs with full-atom pockets of configs[2] size
COND_SEED, JOINT_SEED = 123, 321


# ---- models and inputs ----------------------------------------------------------------------------------------------
def make_ddpm(cfg, joint, timesteps=T, weight_seed=0):
    """The production sampler: synthetic weights, polynomial_2 schedule (precision 5e-4), norm_values (1, 4), the default
    math mode ('auto': 3xFP16 at these widths), deterministic mode, loop engine 'auto' (the graph engine on CUDA)."""
    dyn = EGNNDynamics.from_config(cfg, device='cuda')
    dyn.load_state_dict(syn.synthetic_state_dict(cfg, weight_seed))
    dyn.eval()
    dyn.math_mode = 'auto'
    dyn.deterministic = True
    cls = EnVariationalDiffusion if joint else ConditionalDDPM
    ddpm = cls(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=timesteps,
               noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2', norm_values=(1, 4),
               size_histogram=HIST)
    return ddpm.cuda().eval()


def full_pocket(cfg=FULLATOM_COND):
    """The configs[2] pocket batch (the same one the deterministic sampling test uses) and the ligand sizes."""
    data = syn.synthetic_complex_batch(cfg, COND_LIG, COND_POC, seed=3)
    return ({'x': data['pocket_coords'].cuda(), 'one_hot': data['pocket_one_hot'].cuda(),
             'size': data['num_pocket_nodes'].cuda(), 'mask': data['pocket_mask'].cuda()},
            torch.tensor(COND_LIG).cuda())


# ---- recorder -------------------------------------------------------------------------------------------------------
def _new_record():
    return dict(step=[], z=[], pocket=[], noise=[], t=[], coef3=[], calls=0)


def _replay_recording(rec, st, g, zk, pk, noise_of):
    rec['step'].append(int(st['step']))
    rec['z'].append(st[zk].clone())
    rec['pocket'].append(st[pk].clone())
    g.replay()
    rec['noise'].append(noise_of(st))
    rec['t'].append(st['t'].clone())
    rec['coef3'].append(st['coef3'].clone())


def record_conditional(ddpm, pocket, n_lig, seed=COND_SEED):
    """One seeded ``sample_given_pocket`` call (return_frames=1) with every reverse step recorded."""
    rec = _new_record()

    def steps(z_lig, xh_pocket, lig_mask, pocket_mask, n_samples, first_s, n_steps, timesteps):
        # ConditionalDDPM._graphed_reverse_steps, with the static buffers copied around every replay
        dyn = ddpm.dynamics
        st = ddpm._engine(z_lig, xh_pocket, lig_mask, pocket_mask, n_samples, timesteps)
        prev_defer, dyn.defer_status_check = dyn.defer_status_check, True
        try:
            g = ddpm._graph(st, 'reverse', z_lig, xh_pocket, first_s)
            st['z'].copy_(z_lig); st['pocket'].copy_(xh_pocket); st['step'].fill_(first_s)
            for _ in range(n_steps):
                _replay_recording(rec, st, g, 'z', 'pocket', lambda s: s['noise'].clone())
        finally:
            dyn.defer_status_check = prev_defer
        dyn.check_status()
        rec['calls'] += 1
        rec['z'].append(st['z'].clone()); rec['pocket'].append(st['pocket'].clone())
        rec['lig_mask'], rec['pocket_mask'] = st['lig_mask'].clone(), st['pocket_mask'].clone()
        return st['z'].clone(), st['pocket'].clone()

    ddpm._graphed_reverse_steps = steps
    try:
        torch.manual_seed(seed)
        rec['out'] = ddpm.sample_given_pocket({k: v.clone() for k, v in pocket.items()}, n_lig)
    finally:
        del ddpm._graphed_reverse_steps
    assert rec['calls'] == 1
    return rec


def record_joint(ddpm, n_lig, n_poc, seed=JOINT_SEED):
    """One seeded joint ``sample`` call (return_frames=1) with every reverse step recorded."""
    rec = _new_record()

    def steps(z_lig, z_pocket, lig_mask, pocket_mask, n_samples, first_s, n_steps, timesteps):
        # EnVariationalDiffusion._graphed_joint_reverse_steps, with the static buffers copied around every replay
        dyn = ddpm.dynamics
        st = ddpm._joint_engine(z_lig, z_pocket, lig_mask, pocket_mask, n_samples, timesteps, 1)
        prev_defer, dyn.defer_status_check = dyn.defer_status_check, True
        try:
            g = ddpm._joint_graph(st, 'reverse', z_lig, z_pocket, first_s)
            st['zl'].copy_(z_lig); st['zp'].copy_(z_pocket); st['step'].fill_(first_s)
            for _ in range(n_steps):
                _replay_recording(rec, st, g, 'zl', 'zp', lambda s: tuple(x.clone() for x in s['n_rev']))
        finally:
            dyn.defer_status_check = prev_defer
        dyn.check_status()
        rec['calls'] += 1
        rec['z'].append(st['zl'].clone()); rec['pocket'].append(st['zp'].clone())
        rec['lig_mask'], rec['pocket_mask'] = st['lig_mask'].clone(), st['pocket_mask'].clone()
        return st['zl'].clone(), st['zp'].clone()

    ddpm._graphed_joint_reverse_steps = steps
    try:
        torch.manual_seed(seed)
        rec['out'] = ddpm.sample(len(n_lig), n_lig, n_poc, device='cuda')
    finally:
        del ddpm._graphed_joint_reverse_steps
    assert rec['calls'] == 1
    return rec


# ---- the fused updates and their torch-op references ----------------------------------------------------------------
def ligand_update(ddpm, z, eps, noise, coef3, pocket, lm, pm):
    """dsb_ddpm_ligand_update out of place: (z / c0 - c1 eps + c2 noise, ligand COM removed from ligand and pocket)."""
    z_out, p_out = torch.empty_like(z), torch.empty_like(pocket)
    _native.check(_native.load().dsb_ddpm_ligand_update(
        z.data_ptr(), eps.data_ptr(), noise.data_ptr(), coef3.data_ptr(), lm.data_ptr(), pm.data_ptr(), pocket.data_ptr(),
        z.shape[0], pocket.shape[0], coef3.shape[0], ddpm.atom_nf, ddpm.residue_nf, z_out.data_ptr(), p_out.data_ptr(),
        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return z_out, p_out


def ligand_update_ref(z, eps, noise, coef3, pocket, lm, pm, dtype):
    """The eager reverse step's ops (sample_p_zs_given_zt + sample_normal_zero_com) in ``dtype``."""
    z, eps, noise, coef3, pocket = (x.to(dtype) for x in (z, eps, noise, coef3, pocket))
    out = z / coef3[lm, 0:1] - coef3[lm, 1:2] * eps + coef3[lm, 2:3] * noise
    com = scatter_mean(out[:, :3], lm)
    out[:, :3] -= com[lm]
    p = pocket.clone()
    p[:, :3] -= com[pm]
    return out, p


def joint_update(ddpm, zl, zp, eps_l, eps_p, noise, coef3, lm, pm):
    """dsb_ddpm_joint_update on copies of (zl, zp)."""
    a, b = zl.clone(), zp.clone()
    nx, nhl, nhp = noise
    P = lambda x: x.data_ptr()
    _native.check(_native.load().dsb_ddpm_joint_update(
        P(a), P(b), P(eps_l), P(eps_p), P(nx), P(nhl), P(nhp), P(coef3), P(lm), P(pm), zl.shape[0], zp.shape[0],
        coef3.shape[0], ddpm.atom_nf, ddpm.residue_nf, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return a, b


def joint_update_ref(zl, zp, eps_l, eps_p, noise, coef3, lm, pm, dtype):
    """The eager joint reverse step's ops (sample_p_zs_given_zt: COM-free position noise, mu + sigma eps, joint COM
    projection) in ``dtype``."""
    zl, zp, eps_l, eps_p, coef3 = (x.to(dtype) for x in (zl, zp, eps_l, eps_p, coef3))
    nx, nhl, nhp = (x.to(dtype) for x in noise)
    cm = torch.cat((lm, pm))
    NL = zl.shape[0]
    ex = nx - scatter_mean(nx, cm)[cm]
    wl = zl / coef3[lm, 0:1] - coef3[lm, 1:2] * eps_l + coef3[lm, 2:3] * torch.cat((ex[:NL], nhl), 1)
    wp = zp / coef3[pm, 0:1] - coef3[pm, 1:2] * eps_p + coef3[pm, 2:3] * torch.cat((ex[NL:], nhp), 1)
    mean = scatter_mean(torch.cat((wl[:, :3], wp[:, :3])), cm)
    wl[:, :3] -= mean[lm]
    wp[:, :3] -= mean[pm]
    return wl, wp


# ---- cut-off decisions from float64 distances -----------------------------------------------------------------------
def ulp32(x):
    """Spacing of float32 numbers at |x| (x >= its binade's lower end): 2^(floor(log2 x) - 23)."""
    return 2.0 ** (math.floor(math.log2(abs(x))) - 23)


def candidate_pairs(lm, pm):
    """Every ordered same-graph node pair (i, j) of the global node order [ligand | pocket], self-pairs included (the
    reference's cdist <= cut-off keeps them), with its block: 0 ligand-ligand, 1 pocket-pocket, 2 ligand-pocket or
    pocket-ligand."""
    NL = lm.shape[0]
    mask = torch.cat((lm, pm))
    order = torch.argsort(mask, stable=True)
    counts = torch.bincount(mask)
    rows, cols = [], []
    start = 0
    for n in counts.tolist():
        idx = order[start:start + n]
        rows.append(idx.repeat_interleave(n))
        cols.append(idx.repeat(n))
        start += n
    row, col = torch.cat(rows), torch.cat(cols)
    lig_r, lig_c = row < NL, col < NL
    block = torch.full_like(row, 2)
    block[lig_r & lig_c] = 0
    block[~lig_r & ~lig_c] = 1
    return row, col, block


def pair_distances64(x_lig, x_pocket, row, col):
    """float64 distances of the given pairs, from the float32 coordinates (differences, squares and sum in float64)."""
    x = torch.cat((x_lig, x_pocket)).double()
    return (x[row] - x[col]).pow(2).sum(1).sqrt()


def block_cutoffs(cfg, block, dtype=torch.float64):
    """Per-pair cut-off (inf where the block has none)."""
    cuts = torch.tensor([c if c is not None else math.inf for c in
                         (cfg.edge_cutoff_ligand, cfg.edge_cutoff_pocket, cfg.edge_cutoff_interaction)], dtype=dtype)
    return cuts.to(block.device)[block]


def edge_keys(edges, n):
    return edges[0] * n + edges[1]


def compare_edges(cfg, edges, x_lig, x_pocket, lm, pm, pairs=None, delta_ulps=4):
    """Native edge list against float64 decisions.  Returns (n_checked, n_in_band, n_in_band_disagree, mismatches), where
    mismatches are candidate pairs more than delta_ulps ulp(cut) from their cut-off on which the edge list and the float64
    decision d <= cut disagree.  Also checks that the edge list is sorted, free of duplicates and within graphs."""
    row, col, block = pairs if pairs is not None else candidate_pairs(lm, pm)
    N = lm.shape[0] + pm.shape[0]
    keys = edge_keys(edges, N)
    assert bool((keys[1:] > keys[:-1]).all()), 'edge list not sorted by (row, col) or has duplicates'
    cand = row * N + col
    kept = torch.isin(cand, keys)
    assert int(kept.sum()) == keys.numel(), 'edge list holds pairs of different graphs'
    d = pair_distances64(x_lig, x_pocket, row, col)
    cut = block_cutoffs(cfg, block).to(d.device)
    finite = torch.isfinite(cut)
    ulp = torch.where(finite, torch.exp2(torch.floor(torch.log2(torch.where(finite, cut, 1.0))) - 23), 0.0)
    band = finite & ((d - cut).abs() <= delta_ulps * ulp)
    want = ~finite | (d <= cut)
    bad = ~band & (kept != want)
    return (int(cand.numel()), int(band.sum()), int((band & (kept != want)).sum()),
            [(int(row[i]), int(col[i]), float(d[i]), float(cut[i])) for i in torch.nonzero(bad).flatten()[:10].tolist()])


# ---- planted boundary pairs -----------------------------------------------------------------------------------------
PLANT_CFG = DynamicsConfig(hidden_nf=64, joint_nf=16, n_layers=2, edge_cutoff_ligand=3.0, edge_cutoff_pocket=4.0,
                           edge_cutoff_interaction=7.0)
BLOCKS = ('LL', 'PP', 'LP')
OFFSETS = (-256, -16, -4, -2, -1, 1, 2, 4, 16, 256)     # ulp(cut); +-1 is nextafter(cut, +-inf)
# exact boundary pairs off the axes: integer vectors of length 3 and 7 (for the cut-off 4 only the axis vector exists)
EXACT_VECTORS = {3.0: (1.0, 2.0, 2.0), 4.0: (0.0, 4.0, 0.0), 7.0: (2.0, 3.0, 6.0)}
N_DIRECTIONS = 4


def _cut_of(cfg, blk):
    return {'LL': cfg.edge_cutoff_ligand, 'PP': cfg.edge_cutoff_pocket, 'LP': cfg.edge_cutoff_interaction}[blk]


def _offset_value(cut, k):
    """float32 cut + k ulp(cut) (nextafter steps; below a power of two the steps are the lower binade's)."""
    v = np.float32(cut)
    step = np.float32(np.inf if k > 0 else -np.inf)
    for _ in range(abs(k)):
        v = np.nextafter(v, step)
    return float(v)


def _float32_neighbours(v, n=4):
    """v and its n float32 neighbours on either side."""
    out = [np.float32(v)]
    for step in (np.float32(-np.inf), np.float32(np.inf)):
        w = np.float32(v)
        for _ in range(n):
            w = np.nextafter(w, step)
            out.append(w)
    return np.array(out, dtype=np.float32)


def _generic_pair(rng, cut, target):
    """float32 points p, q with |p| in [10, 30] A and a float64 |p - q| within ulp(cut) / 8 of ``target``: q is the best
    of the 9^3 float32 points around the rounded p + target * u.  On most draws one coordinate of p is near zero and the
    pair straddles it, so that the float32 difference of that coordinate rounds."""
    while True:
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        v = rng.normal(size=3)
        p = (v / np.linalg.norm(v) * rng.uniform(10.0, 30.0)).astype(np.float32)
        if rng.uniform() < 0.75:
            ax = rng.integers(3)
            p[ax] = np.float32(rng.uniform(-1.0, 1.0) * (1e-3 if rng.uniform() < 0.5 else 1.0))
            u[ax] = abs(u[ax]) + 0.5
            u /= np.linalg.norm(u)
        if not 10.0 <= np.linalg.norm(p.astype(np.float64)) <= 30.0:
            continue
        q0 = (p.astype(np.float64) + target * u).astype(np.float32)
        axes = [_float32_neighbours(q0[a]) for a in range(3)]
        cand = np.stack(np.meshgrid(*axes, indexing='ij'), -1).reshape(-1, 3)
        d = np.sqrt(((cand.astype(np.float64) - p.astype(np.float64)) ** 2).sum(1))
        i = int(np.argmin(np.abs(d - target)))
        if abs(d[i] - target) <= 0.125 * ulp32(cut):
            return p, cand[i]


def planted_batch(cfg=PLANT_CFG, seed=0):
    """Denoiser inputs (CPU) with one planted pair per graph, and the list of pairs: dict(block, kind ('exact_axis',
    'exact_far', 'axis', 'generic'), k (ulp offset, 0 = exactly at the cut-off), cut, claimed (float64 distance the pair is
    built to have), graph, i, j (global node indices in [ligand | pocket] order))."""
    rng = np.random.default_rng(seed)
    graphs = []                  # (block, kind, k, cut, claimed, p, q)
    for blk in BLOCKS:
        cut = float(_cut_of(cfg, blk))
        graphs.append((blk, 'exact_axis', 0, cut, cut, np.array([0.0, 1.5, -2.0], np.float32),
                       np.array([cut, 1.5, -2.0], np.float32)))
        base = np.array([12.5, -17.25, 21.0], np.float32)
        graphs.append((blk, 'exact_far', 0, cut, cut, base, base + np.array(EXACT_VECTORS[cut], np.float32)))
        for k in OFFSETS:
            c = _offset_value(cut, k)
            graphs.append((blk, 'axis', k, cut, c, np.array([0.0, -0.75, 2.25], np.float32),
                           np.array([c, -0.75, 2.25], np.float32)))
            for _ in range(N_DIRECTIONS):
                p, q = _generic_pair(rng, cut, c)
                graphs.append((blk, 'generic', k, cut, c, p, q))
    lig_x, lig_g, poc_x, poc_g, meta = [], [], [], [], []
    for g, (blk, kind, k, cut, claimed, p, q) in enumerate(graphs):
        if blk == 'LL':
            lig_x += [p, q]; lig_g += [g, g]
        elif blk == 'PP':
            poc_x += [p, q]; poc_g += [g, g]
        else:
            lig_x.append(p); lig_g.append(g)
            poc_x.append(q); poc_g.append(g)
        meta.append(dict(block=blk, kind=kind, k=k, cut=cut, claimed=claimed, graph=g))
    NL = len(lig_x)
    lm, pm = torch.tensor(lig_g), torch.tensor(poc_g)
    for m in meta:
        g = m['graph']
        li = torch.nonzero(lm == g).flatten().tolist()
        pi = [NL + i for i in torch.nonzero(pm == g).flatten().tolist()]
        m['i'], m['j'] = (li + pi)[0], (li + pi)[1]
    gen = torch.Generator().manual_seed(seed)
    A, R = cfg.atom_nf, cfg.residue_nf
    h_l = torch.nn.functional.one_hot(torch.randint(0, A, (NL,), generator=gen), A).float() / 4
    h_p = torch.nn.functional.one_hot(torch.randint(0, R, (len(poc_x),), generator=gen), R).float() / 4
    xh_l = torch.cat((torch.from_numpy(np.stack(lig_x)), h_l), 1)
    xh_p = torch.cat((torch.from_numpy(np.stack(poc_x)), h_p), 1)
    t = torch.rand((len(graphs), 1), generator=gen)
    return (xh_l, xh_p, t, lm, pm), meta
