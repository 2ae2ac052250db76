"""Cost of the deterministic mode at configs[2]: full-atom conditional model (hidden_nf 256, 6 layers), batch 64 of 25 ligand
atoms + 175 pocket nodes.

For each math mode ('3xfp16', 'fp32') the two modes are timed alternately in one process after warm-up:
* one denoiser call (CUDA events over --calls calls per round, --rounds rounds), and its split by kernel class from the
  library's profiling hook (dsb_dynamics_set_profiling; the segment reduces of the deterministic mode count under
  edge_gcl / edge_coord);
* one 500-step ConditionalDDPM.sample_given_pocket run on the CUDA-graph loop engine (--sample-rounds rounds).
Prints one JSON line with the GPU name and power limit read in the same run.  Needs a CUDA device.

    python profiles/deterministic_overhead.py [--calls 50] [--rounds 5] [--sample-rounds 2] [--out result.json]
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

from diffsbdd_b200 import synthetic as syn  # noqa: E402
from diffsbdd_b200.conditional_model import ConditionalDDPM  # noqa: E402
from diffsbdd_b200.config import FULLATOM_COND  # noqa: E402
from diffsbdd_b200.dynamics import EGNNDynamics  # noqa: E402

B, N_LIG, N_POCKET, T = 64, 25, 175, 500
MODES = {False: 'default', True: 'deterministic'}


def power_limit_w():
    try:
        out = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except Exception:  # noqa: BLE001
        return None


def time_ms(fn, n):
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(n):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--calls', type=int, default=50)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--sample-rounds', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('deterministic_overhead.py needs a CUDA device')
    cfg = FULLATOM_COND
    sd = syn.synthetic_state_dict(cfg, 0)
    dyn = EGNNDynamics.from_config(cfg, device='cuda')
    dyn.load_state_dict(sd)
    dyn.eval()
    inp = [x.cuda() for x in syn.synthetic_denoiser_inputs(cfg, [N_LIG] * B, [N_POCKET] * B, seed=1)]
    ddpm = ConditionalDDPM(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=T,
                           noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2', norm_values=(1, 4),
                           size_histogram=[[1.0] * (N_POCKET + 2)] * (N_LIG + 2)).cuda().eval()
    ddpm.loop_engine = 'graph'
    data = syn.synthetic_complex_batch(cfg, [N_LIG] * B, [N_POCKET] * B, seed=3)
    pocket = {'x': data['pocket_coords'].cuda(), 'one_hot': data['pocket_one_hot'].cuda(),
              'size': data['num_pocket_nodes'].cuda(), 'mask': data['pocket_mask'].cuda()}
    n_lig = torch.full((B,), N_LIG, device='cuda')

    res = {'workload': 'deterministic_overhead', 'config': 'configs[2] crossdock_fullatom_cond', 'batch': B, 'n_lig': N_LIG,
           'n_pocket': N_POCKET, 'hidden_nf': cfg.hidden_nf, 'n_layers': cfg.n_layers,
           'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit_w(), 'calls_per_round': args.calls,
           'rounds': args.rounds}
    with torch.no_grad():
        for mm in ('3xfp16', 'fp32'):
            dyn.math_mode = mm
            call_ms = {False: [], True: []}
            launches, ws_bytes, by_class = {}, {}, {}
            for det in (False, True):                                   # warm-up: workspace, plan cache, clocks
                dyn.deterministic = det
                time_ms(lambda: dyn(*inp), 10)
                launches[det], ws_bytes[det] = dyn.launches_per_forward, dyn._workspace.numel()
            for _ in range(args.rounds):
                for det in (False, True):
                    dyn.deterministic = det
                    call_ms[det].append(time_ms(lambda: dyn(*inp), args.calls))
            for det in (False, True):                                   # per-class split (events between kernels)
                dyn.deterministic = det
                dyn.set_profiling(True)
                dyn.collect_profile(reset=True)
                time_ms(lambda: dyn(*inp), args.calls)
                prof = dyn.collect_profile(reset=True)
                dyn.set_profiling(False)
                by_class[det] = {k: round(v['ms'] / args.calls, 4) for k, v in prof.items()}
            sample_s = {False: [], True: []}
            for r in range(args.sample_rounds + 1):                      # round 0 captures the graphs: not timed
                for det in (False, True):
                    dyn.deterministic = det
                    torch.manual_seed(0)
                    torch.cuda.synchronize()
                    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    start.record()
                    ddpm.sample_given_pocket({k: v.clone() for k, v in pocket.items()}, n_lig)
                    end.record()
                    torch.cuda.synchronize()
                    if r > 0:
                        sample_s[det].append(start.elapsed_time(end) / 1000.0)
            for det, name in MODES.items():
                res[f'{mm}_{name}_call_ms_median'] = statistics.median(call_ms[det])
                res[f'{mm}_{name}_call_ms_rounds'] = [round(x, 4) for x in call_ms[det]]
                res[f'{mm}_{name}_ms_by_class'] = by_class[det]
                res[f'{mm}_{name}_launches'] = launches[det]
                res[f'{mm}_{name}_workspace_mb'] = round(ws_bytes[det] / 2 ** 20, 1)
                res[f'{mm}_{name}_sample500_s'] = [round(x, 3) for x in sample_s[det]]
            res[f'{mm}_call_overhead'] = (res[f'{mm}_deterministic_call_ms_median'] /
                                          res[f'{mm}_default_call_ms_median'] - 1.0)
            res[f'{mm}_sample500_overhead'] = statistics.median(sample_s[True]) / statistics.median(sample_s[False]) - 1.0
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
