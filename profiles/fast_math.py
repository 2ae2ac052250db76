"""What the single-product math mode ('1xfp16', 31) buys over the default tensor-core mode ('3xfp16', 15).

For bench.py's `fullatom` (configs[2]), `inpaint`, `moad`, `ca` and `moad_ca` shapes (synthetic weights and pockets, batch
and sizes of bench.py's WORKLOADS), modes 15 and 31 alternate in one process:
  * per denoiser call, the time of each kernel class (dsb_dynamics_set_profiling: CUDA events around the launches of each
    class, eager forwards, each after bench.py's L2 flush) and the number of node-GEMM launches;
  * one 500-step sampling run on the CUDA-graph loop engine (`sample_given_pocket`; `inpaint`: ConditionalDDPM.inpaint
    with 500 steps and one resampling, 10 fixed atoms), as ligand atoms / s; round 0 captures the graphs and is not timed.
The card's name, power limit and SM clocks are read in the same run.  Prints one JSON line.  Needs a CUDA device.

    python profiles/fast_math.py [--shapes fullatom,inpaint,moad,ca,moad_ca] [--rounds 3] [--calls 20] [--out f.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from diffsbdd_b200 import synthetic as syn  # noqa: E402
from diffsbdd_b200.conditional_model import ConditionalDDPM  # noqa: E402
from diffsbdd_b200.dynamics import EGNNDynamics  # noqa: E402

T = 500
MODES = ('3xfp16', '1xfp16')


def gpu_info():
    out = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
    return out


def build(shape):
    a = argparse.Namespace(workload=shape, n_fixed=10)
    cfg, density, norm_values, _ = bench.workload(a)
    _, B, NL, NP, _, _, _, _ = bench.WORKLOADS[shape]
    dyn = EGNNDynamics.from_config(cfg, device='cuda')
    dyn.load_state_dict(syn.synthetic_state_dict(cfg, 0))
    dyn.eval()
    ddpm = ConditionalDDPM(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=T,
                           noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2', norm_values=norm_values,
                           size_histogram=[[1.0] * (NP + 2)] * (NL + 2)).cuda().eval()
    ddpm.loop_engine = 'graph'
    pocket = {k: v.cuda() for k, v in syn.synthetic_pocket(cfg, [NP] * B, seed=3, density=density).items()}
    n_lig = torch.full((B,), NL, dtype=torch.int64, device='cuda')
    if shape == 'inpaint':
        lig, fixed = bench.inpaint_inputs(cfg, argparse.Namespace(n_lig=NL, n_fixed=10), B, 3, 'cuda')

        def run():
            return ddpm.inpaint({k: v.clone() for k, v in lig.items()}, {k: v.clone() for k, v in pocket.items()}, fixed,
                                resamplings=1, timesteps=T, center='ligand')
    else:
        def run():
            return ddpm.sample_given_pocket({k: v.clone() for k, v in pocket.items()}, n_lig)
    inp = [x.cuda() for x in syn.synthetic_denoiser_inputs(cfg, [NL] * B, [NP] * B, seed=1)]
    return cfg, dyn, run, inp, B * NL


def per_call(dyn, inp, calls, flush):
    """ms per call of each kernel class, and the node-GEMM launches of one call."""
    with torch.no_grad():
        dyn(*inp)
        dyn.set_profiling(True)
        dyn.collect_profile(reset=True)
        for _ in range(calls):
            bench.l2_flush(flush)
            dyn(*inp)
        prof = dyn.collect_profile(reset=True)
        dyn.set_profiling(False)
    torch.cuda.synchronize()
    out = {k: round(v['ms'] / calls, 4) for k, v in prof.items()}
    out['node_gemm_launches'] = prof['node_gemm']['intervals'] // calls
    out['launches'] = dyn.launches_per_forward
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--shapes', default='fullatom,inpaint,moad,ca,moad_ca')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('fast_math.py needs a CUDA device')
    flush = torch.zeros(64 * 1024 * 1024, dtype=torch.float32, device='cuda')
    res = {'profile': 'fast_math', 'gpu': gpu_info(), 'steps': T, 'rounds': args.rounds, 'shapes': {}}
    for shape in args.shapes.split(','):
        cfg, dyn, run, inp, atoms = build(shape)
        r = {'hidden_nf': cfg.hidden_nf, 'ligand_atoms': atoms}
        times = {m: [] for m in MODES}
        for rd in range(args.rounds + 1):
            for m in MODES:
                dyn.math_mode = m
                torch.manual_seed(0)
                torch.cuda.synchronize()
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                run()
                end.record()
                torch.cuda.synchronize()
                if rd > 0:
                    times[m].append(start.elapsed_time(end) / 1000.0)
        for m in MODES:
            dyn.math_mode = m
            r[m] = {'sample_s': [round(x, 3) for x in times[m]],
                    'ligand_atoms_per_s': round(atoms / statistics.median(times[m]), 1),
                    'per_call_ms': per_call(dyn, inp, args.calls, flush)}
        r['speedup'] = round(statistics.median(times['3xfp16']) / statistics.median(times['1xfp16']), 3)
        res['shapes'][shape] = r
        print(shape, json.dumps(r), file=sys.stderr, flush=True)
        del dyn, run
        torch.cuda.empty_cache()
    res['gpu_after'] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
