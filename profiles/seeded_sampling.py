"""Cost of seeded sampling (``seeds=``) at configs[2]: full-atom conditional model (hidden_nf 256, 6 layers, 3xFP16), batch
64 of 25 ligand atoms + 175 pocket nodes, one 500-step ConditionalDDPM.sample_given_pocket run on the CUDA-graph loop
engine.  Seeded and unseeded runs alternate, in the default and the deterministic mode; round 0 captures the graphs and is
not timed.  Prints one JSON line with the GPU name and power limit read in the same run.  Needs a CUDA device.

    python profiles/seeded_sampling.py [--rounds 3] [--out result.json]
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
sys.path.insert(0, os.path.join(ROOT, 'profiles'))

from deterministic_overhead import B, N_LIG, N_POCKET, T, power_limit_w  # noqa: E402
from diffsbdd_b200 import synthetic as syn  # noqa: E402
from diffsbdd_b200.conditional_model import ConditionalDDPM  # noqa: E402
from diffsbdd_b200.config import FULLATOM_COND  # noqa: E402
from diffsbdd_b200.dynamics import EGNNDynamics  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('seeded_sampling.py needs a CUDA device')
    cfg = FULLATOM_COND
    dyn = EGNNDynamics.from_config(cfg, device='cuda')
    dyn.load_state_dict(syn.synthetic_state_dict(cfg, 0))
    dyn.eval()
    dyn.math_mode = '3xfp16'
    ddpm = ConditionalDDPM(dynamics=dyn, atom_nf=cfg.atom_nf, residue_nf=cfg.residue_nf, n_dims=3, timesteps=T,
                           noise_schedule='polynomial_2', noise_precision=5e-4, loss_type='l2', norm_values=(1, 4),
                           size_histogram=[[1.0] * (N_POCKET + 2)] * (N_LIG + 2)).cuda().eval()
    ddpm.loop_engine = 'graph'
    data = syn.synthetic_complex_batch(cfg, [N_LIG] * B, [N_POCKET] * B, seed=3)
    pocket = {'x': data['pocket_coords'].cuda(), 'one_hot': data['pocket_one_hot'].cuda(),
              'size': data['num_pocket_nodes'].cuda(), 'mask': data['pocket_mask'].cuda()}
    n_lig = torch.full((B,), N_LIG, device='cuda')
    seeds = torch.arange(B)
    variants = [(det, sd) for det in (False, True) for sd in (False, True)]
    times = {v: [] for v in variants}
    for r in range(args.rounds + 1):
        for det, sd in variants:
            dyn.deterministic = det
            torch.manual_seed(0)
            torch.cuda.synchronize()
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            ddpm.sample_given_pocket({k: v.clone() for k, v in pocket.items()}, n_lig, seeds=seeds if sd else None)
            end.record()
            torch.cuda.synchronize()
            if r > 0:
                times[(det, sd)].append(start.elapsed_time(end) / 1000.0)
    res = {'workload': 'seeded_sampling', 'config': 'configs[2] crossdock_fullatom_cond 3xfp16', 'batch': B, 'steps': T,
           'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit_w(), 'rounds': args.rounds}
    for det in (False, True):
        m = 'deterministic' if det else 'default'
        for sd in (False, True):
            res[f'{m}_{"seeded" if sd else "unseeded"}_sample500_s'] = [round(x, 3) for x in times[(det, sd)]]
        res[f'{m}_seeded_overhead'] = statistics.median(times[(det, True)]) / statistics.median(times[(det, False)]) - 1.0
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
