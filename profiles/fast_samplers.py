"""What the few-step samplers buy: 500-step 'ddpm' against 'ddim' (eta = 0) and 'dpmpp_2m' at N = 50, 100 and 250 steps.

For bench.py's `fullatom` (configs[2]) and `moad` shapes (synthetic weights and pockets, batch and sizes of bench.py's
WORKLOADS), in the math modes '3xfp16' and '1xfp16': one ConditionalDDPM per arm (sampler, N), all sharing one native
denoiser, so that every arm keeps its own captured CUDA-graph step; the arms alternate within each round, and round 0
captures and is not timed.  Each timed run is one whole `sample_given_pocket` call on the graph engine (prior, N replays,
the t = 0 call), timed with CUDA events; reported as ligand atoms / s and as ms per denoiser call (run time / (N + 1)).
The card's name, power limit and SM clocks are read in the same run.  Prints one JSON line.  Needs a CUDA device.
Sample quality is not measured here: synthetic weights say nothing about it.

    python profiles/fast_samplers.py [--shapes fullatom,moad] [--rounds 2] [--out f.json]
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
MODES = ('3xfp16', '1xfp16')
ARMS = [('ddpm', T)] + [(s, n) for s in ('ddim', 'dpmpp_2m') for n in (50, 100, 250)]


def build(shape):
    a = argparse.Namespace(workload=shape, n_fixed=10)
    cfg, density, norm_values, _ = bench.workload(a)
    _, B, NL, NP, _, _, _, _ = bench.WORKLOADS[shape]
    dyn = EGNNDynamics.from_config(cfg, device='cuda')
    dyn.load_state_dict(syn.synthetic_state_dict(cfg, 0))
    dyn.eval()
    pocket = {k: v.cuda() for k, v in syn.synthetic_pocket(cfg, [NP] * B, seed=3, density=density).items()}
    n_lig = torch.full((B,), NL, dtype=torch.int64, device='cuda')
    runs = {}
    for sampler, n in ARMS:
        ddpm = ConditionalDDPM(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=T,
                               noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2', norm_values=norm_values,
                               size_histogram=[[1.0] * (NP + 2)] * (NL + 2)).cuda().eval()
        ddpm.loop_engine = 'graph'
        runs[f'{sampler}_{n}'] = (lambda d=ddpm, s=sampler, k=n: d.sample_given_pocket(
            {key: v.clone() for key, v in pocket.items()}, n_lig, timesteps=k, sampler=s), n)
    return cfg, dyn, runs, B * NL


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default='fullatom,moad')
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('fast_samplers.py needs a CUDA device')
    res = {'profile': 'fast_samplers', 'gpu': gpu_info(), 'rounds': args.rounds, 'shapes': {}}
    for shape in args.shapes.split(','):
        cfg, dyn, runs, atoms = build(shape)
        r = {'hidden_nf': cfg.hidden_nf, 'ligand_atoms': atoms}
        for m in MODES:
            dyn.math_mode = m
            times = {k: [] for k in runs}
            for rd in range(args.rounds + 1):
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
            base = statistics.median(times[f'ddpm_{T}'])
            r[m] = {k: {'sample_s': [round(x, 3) for x in v],
                        'ligand_atoms_per_s': round(atoms / statistics.median(v), 1),
                        'ms_per_call': round(1000.0 * statistics.median(v) / (runs[k][1] + 1), 3),
                        'speedup_vs_ddpm_500': round(base / statistics.median(v), 2)} for k, v in times.items()}
        res['shapes'][shape] = r
        print(shape, json.dumps(r), file=sys.stderr, flush=True)
        del dyn, runs
        torch.cuda.empty_cache()
    res['gpu_after'] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
