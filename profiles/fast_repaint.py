"""What the few-step samplers buy on the RePaint paths (DESIGN §14): inpainting, joint-model generation for a fixed pocket and
diversify, each ancestral ('ddpm') against 'ddim' (eta = 0) and 'dpmpp_2m' on fewer steps.

* inpaint: bench.py's `inpaint` shape (64 x (25 + 175), 10 fixed atoms, center='ligand'): ancestral 50 x 20 resamplings
  against the few-step samplers at 10 x 20 and 25 x 20;
* joint: the joint full-atom model at the same shape generating with every pocket node fixed (EnVariationalDiffusion.inpaint,
  resamplings 1): 500 ancestral steps against 50 few-step steps;
* diversify: the `inpaint` shape, noising_steps 100 of T = 500: the ancestral 100 steps against 10 and 20 few-step steps.

3xFP16 math mode, CUDA-graph engine, synthetic weights.  One model object per arm, all sharing one native denoiser per shape,
so each arm keeps its captured steps; the arms alternate within each round, and round 0 captures and is not timed.  Each
timed run is one whole sampler call timed with CUDA events, reported as ligand atoms / s and ms per denoiser call (run time
/ calls).  The card's name, power limit and SM clock are read in the same run.  Prints one JSON line.  Needs a CUDA device.
Sample quality is not measured: synthetic weights say nothing about it.

    python profiles/fast_repaint.py [--rounds 2] [--out f.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from diffsbdd_b200 import synthetic as syn  # noqa: E402
from diffsbdd_b200.conditional_model import ConditionalDDPM  # noqa: E402
from diffsbdd_b200.config import FULLATOM_JOINT  # noqa: E402
from diffsbdd_b200.dynamics import EGNNDynamics  # noqa: E402
from diffsbdd_b200.en_diffusion import EnVariationalDiffusion  # noqa: E402
from profiles.fast_math import gpu_info  # noqa: E402

T = 500
FAST = ('ddim', 'dpmpp_2m')


def _model(cls, cfg, dyn, norm_values, NL, NP):
    ddpm = cls(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=T,
               noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2', norm_values=norm_values,
               size_histogram=[[1.0] * (NP + 2)] * (NL + 2)).cuda().eval()
    ddpm.loop_engine = 'graph'
    return ddpm


def build():
    """{group: (ligand atoms per run, {arm: (run, denoiser calls)})}."""
    a = argparse.Namespace(workload='inpaint', n_fixed=10)
    cfg, density, norm_values, _ = bench.workload(a)
    _, B, NL, NP, _, _, _, _ = bench.WORKLOADS['inpaint']
    groups = {}
    dyn = EGNNDynamics.from_config(cfg, device='cuda')
    dyn.load_state_dict(syn.synthetic_state_dict(cfg, 0))
    dyn.eval()
    dyn.math_mode = '3xfp16'
    pocket = {k: v.cuda() for k, v in syn.synthetic_pocket(cfg, [NP] * B, seed=3, density=density).items()}
    lig, fixed = bench.inpaint_inputs(cfg, argparse.Namespace(n_lig=NL, n_fixed=10), B, 3, 'cuda')
    copy = lambda d: {k: v.clone() for k, v in d.items()}

    def inpaint(sampler, n):
        d = _model(ConditionalDDPM, cfg, dyn, norm_values, NL, NP)
        return (lambda: d.inpaint(copy(lig), copy(pocket), fixed, resamplings=20, timesteps=n, center='ligand',
                                  sampler=sampler)), n * 20 + 1
    arms = {'ddpm_50x20': inpaint('ddpm', 50)}
    arms.update({f'{s}_{n}x20': inpaint(s, n) for s in FAST for n in (10, 25)})
    groups['inpaint'] = (B * NL, arms)

    def diversify(sampler, k):
        d = _model(ConditionalDDPM, cfg, dyn, norm_values, NL, NP)
        kw = {} if sampler == 'ddpm' else dict(sampler=sampler, denoising_steps=k)
        return (lambda: d.diversify(copy(lig), copy(pocket), 100, **kw)), k + 1
    arms = {'ddpm_100': diversify('ddpm', 100)}
    arms.update({f'{s}_{k}': diversify(s, k) for s in FAST for k in (10, 20)})
    groups['diversify'] = (B * NL, arms)

    jcfg = FULLATOM_JOINT
    jdyn = EGNNDynamics.from_config(jcfg, device='cuda')
    jdyn.load_state_dict(syn.synthetic_state_dict(jcfg, 0))
    jdyn.eval()
    jdyn.math_mode = '3xfp16'
    jpocket = {k: v.cuda() for k, v in syn.synthetic_pocket(jcfg, [NP] * B, seed=3, density=density).items()}
    jlig, _ = bench.inpaint_inputs(jcfg, argparse.Namespace(n_lig=NL, n_fixed=0), B, 3, 'cuda')
    lf, pf = torch.zeros(B * NL, device='cuda'), torch.ones(B * NP, device='cuda')

    def joint(sampler, n):
        d = _model(EnVariationalDiffusion, jcfg, jdyn, norm_values, NL, NP)
        return (lambda: d.inpaint(copy(jlig), copy(jpocket), lf, pf, timesteps=n, sampler=sampler)), n + 1
    arms = {'ddpm_500': joint('ddpm', 500)}
    arms.update({f'{s}_50': joint(s, 50) for s in FAST})
    groups['joint'] = (B * NL, arms)
    return groups


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('fast_repaint.py needs a CUDA device')
    res = {'profile': 'fast_repaint', 'gpu': gpu_info(), 'rounds': args.rounds, 'groups': {}}
    groups = build()
    times = {g: {k: [] for k in arms} for g, (_, arms) in groups.items()}
    failed = {}     # arm -> the error of its run: with synthetic weights a run may leave the fp16 range; it is reported, not timed
    for rd in range(args.rounds + 1):
        for g, (_, arms) in groups.items():
            for k, (run, _) in arms.items():
                if (g, k) in failed:
                    continue
                torch.manual_seed(0)
                torch.cuda.synchronize()
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                try:
                    run()
                except ValueError as e:
                    failed[(g, k)] = str(e)
                    continue
                end.record()
                torch.cuda.synchronize()
                if rd > 0:
                    times[g][k].append(start.elapsed_time(end) / 1000.0)
    for g, (atoms, arms) in groups.items():
        base = statistics.median(times[g][next(iter(arms))]) if times[g][next(iter(arms))] else None
        res['groups'][g] = {}
        for k, v in times[g].items():
            if (g, k) in failed:
                res['groups'][g][k] = {'calls': arms[k][1], 'error': failed[(g, k)]}
                continue
            med = statistics.median(v)
            res['groups'][g][k] = {'calls': arms[k][1], 'run_s': [round(x, 3) for x in v],
                                   'ligand_atoms_per_s': round(atoms / med, 1), 'ms_per_call': round(1000.0 * med / arms[k][1], 3),
                                   'speedup_vs_ancestral': round(base / med, 2) if base else None}
        print(g, json.dumps(res['groups'][g]), file=sys.stderr, flush=True)
    res['gpu_after'] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
