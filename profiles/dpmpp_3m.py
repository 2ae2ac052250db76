"""DPM-Solver++(3M) against 2M: time per denoiser call, and distance from the converged ODE solution.

Speed: 'dpmpp_2m' and 'dpmpp_3m' at N = 20 and 50 steps for bench.py's `fullatom` (configs[2]) and `moad` shapes (synthetic
weights and pockets, batch and sizes of bench.py's WORKLOADS, default math mode, CUDA-graph engine).  One ConditionalDDPM per
arm, all sharing one native denoiser, so every arm keeps its own captured step; the arms alternate within each round, and
round 0 captures and is not timed.  Each timed run is one whole `sample_given_pocket` call, timed with CUDA events; reported
as ligand atoms / s and ms per denoiser call (run time / (N + 1)).

Error: on configs[2] with synthetic weights and the same seeds for every arm (so every arm starts from the same z_T and
ends with the same final draw), the RMS distance of the ligand coordinates (Angstrom) of 2M and 3M samples at N = 10, 20,
25, 50 and 100 from a 500-step 3M solution.  This is distance to the solution of the sampling ODE, not sample quality.

The card's name, power limit and SM clocks are read in the same run.  Prints one JSON line.  Needs a CUDA device.

    python profiles/dpmpp_3m.py [--shapes fullatom,moad] [--rounds 2] [--out f.json]
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
from diffsbdd_b200.dynamics import EGNNDynamics  # noqa: E402
from profiles.fast_math import gpu_info  # noqa: E402

T = 500
SPEED_ARMS = [(s, n) for n in (20, 50) for s in ('dpmpp_2m', 'dpmpp_3m')]
ERROR_STEPS = (10, 20, 25, 50, 100)
REFERENCE_STEPS = 500


def build(shape, arms):
    a = argparse.Namespace(workload=shape, n_fixed=10)
    cfg, density, norm_values, _ = bench.workload(a)
    _, B, NL, NP, _, _, _, _ = bench.WORKLOADS[shape]
    dyn = EGNNDynamics.from_config(cfg, device='cuda')
    dyn.load_state_dict(syn.synthetic_state_dict(cfg, 0))
    dyn.eval()
    pocket = {k: v.cuda() for k, v in syn.synthetic_pocket(cfg, [NP] * B, seed=3, density=density).items()}
    n_lig = torch.full((B,), NL, dtype=torch.int64, device='cuda')
    runs = {}
    for sampler, n in arms:
        ddpm = ConditionalDDPM(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=T,
                               noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2', norm_values=norm_values,
                               size_histogram=[[1.0] * (NP + 2)] * (NL + 2)).cuda().eval()
        ddpm.loop_engine = 'graph'
        runs[f'{sampler}_{n}'] = (lambda d=ddpm, s=sampler, k=n, **kw: d.sample_given_pocket(
            {key: v.clone() for key, v in pocket.items()}, n_lig, timesteps=k, sampler=s, **kw), n)
    return cfg, dyn, runs, B * NL


def speed(shape, rounds):
    cfg, dyn, runs, atoms = build(shape, SPEED_ARMS)
    times = {k: [] for k in runs}
    for rd in range(rounds + 1):
        for k, (run, _) in runs.items():
            torch.manual_seed(0)
            torch.cuda.synchronize()
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            run()
            end.record()
            torch.cuda.synchronize()
            if rd > 0:
                times[k].append(start.elapsed_time(end) / 1000.0)
    return {'hidden_nf': cfg.hidden_nf, 'math_mode': dyn.math_mode, 'ligand_atoms': atoms,
            'arms': {k: {'sample_s': [round(x, 4) for x in v], 'ligand_atoms_per_s': round(atoms / statistics.median(v), 1),
                         'ms_per_call': round(1000.0 * statistics.median(v) / (runs[k][1] + 1), 3)} for k, v in times.items()}}


def error():
    arms = [('dpmpp_3m', REFERENCE_STEPS)] + [(s, n) for n in ERROR_STEPS for s in ('dpmpp_2m', 'dpmpp_3m')]
    _, _, runs, _ = build('fullatom', arms)
    seeds = torch.arange(64) * 7919 + 11
    x = {k: run(seeds=seeds)[0][:, :3].double() for k, (run, _) in runs.items()}
    ref = x[f'dpmpp_3m_{REFERENCE_STEPS}']
    rms = lambda a: float(((a - ref) ** 2).mean().sqrt())
    return {'reference': f'dpmpp_3m_{REFERENCE_STEPS}', 'rms_angstrom': {k: round(rms(v), 5) for k, v in x.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default='fullatom,moad')
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('dpmpp_3m.py needs a CUDA device')
    res = {'profile': 'dpmpp_3m', 'gpu': gpu_info(), 'rounds': args.rounds, 'speed': {}}
    for shape in args.shapes.split(','):
        res['speed'][shape] = speed(shape, args.rounds)
        print(shape, json.dumps(res['speed'][shape]), file=sys.stderr, flush=True)
        torch.cuda.empty_cache()
    res['error'] = error()
    res['gpu_after'] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
