"""Throughput of likelihood evaluation (``LigandPocketDDPM.forward`` in eval mode) at configs[2]: full-atom conditional
model (hidden_nf 256, 6 layers), batch 64, 25 ligand atoms + 175 pocket nodes, 500 diffusion steps.

Times the native path (two native denoiser calls + one fused dsb_ddpm_vlb_terms launch) against the eager path (the same
native denoiser, loss terms as reference-order torch ops) with CUDA events over --batches batches after --warmup warm-ups,
and splits the native forward into its two denoiser calls, the fused terms kernel and the rest.  Prints one JSON line with
the GPU name and power limit read in the same run.  Needs a CUDA device.

    python profiles/nll_throughput.py [--batches 50] [--warmup 5] [--out result.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from argparse import Namespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from diffsbdd_b200 import synthetic as syn  # noqa: E402
from diffsbdd_b200.config import FULLATOM_COND  # noqa: E402
from diffsbdd_b200.lightning_modules import LigandPocketDDPM  # noqa: E402

B, N_LIG, N_POCKET, T = 64, 25, 175, 500


def power_limit_w():
    try:
        out = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except Exception:  # noqa: BLE001
        return None


def build_model(cfg):
    egnn = Namespace(device='cuda', **{k: v for k, v in cfg.kwargs().items()
                                       if k not in ('atom_nf', 'residue_nf', 'n_dims', 'condition_time', 'mode',
                                                    'update_pocket_coords')})
    diff = Namespace(diffusion_steps=T, diffusion_noise_schedule='polynomial_2', diffusion_noise_precision=5.0e-4,
                     diffusion_loss_type='l2', normalize_factors=[1, 4])
    model = LigandPocketDDPM(outdir=None, dataset='crossdock', datadir=None, batch_size=B, lr=1e-3, egnn_params=egnn,
                             diffusion_params=diff, num_workers=0, augment_noise=0, augment_rotation=False, clip_grad=True,
                             eval_epochs=1, eval_params=Namespace(), visualize_sample_epoch=1, visualize_chain_epoch=1,
                             auxiliary_loss=False, loss_params=Namespace(), mode='pocket_conditioning',
                             node_histogram=np.ones((N_LIG + 2, N_POCKET + 2)).tolist(), pocket_representation='full-atom')
    model.ddpm.dynamics.load_state_dict(syn.synthetic_state_dict(cfg, 0))
    return model.to('cuda').eval()


def time_ms(fn, n, warmup):
    for _ in range(warmup):
        fn()
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
    ap.add_argument('--batches', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('nll_throughput.py needs a CUDA device')
    cfg = FULLATOM_COND
    model = build_model(cfg)
    ddpm, dyn = model.ddpm, model.ddpm.dynamics
    data = syn.synthetic_complex_batch(cfg, [N_LIG] * B, [N_POCKET] * B, seed=3)
    data = {k: v.cuda() for k, v in data.items()}
    torch.manual_seed(0)

    res = {'workload': 'nll_eval', 'config': 'configs[2] crossdock_fullatom_cond', 'batch': B, 'n_lig': N_LIG,
           'n_pocket': N_POCKET, 'hidden_nf': cfg.hidden_nf, 'n_layers': cfg.n_layers, 'math_mode': dyn.math_mode,
           'batches_timed': args.batches, 'gpu': torch.cuda.get_device_name(0), 'power_limit_w': power_limit_w()}
    with torch.no_grad():
        for engine in ('auto', 'eager'):
            ddpm.loop_engine = engine
            ms = time_ms(lambda: model(data), args.batches, args.warmup)
            key = 'native' if engine == 'auto' else 'eager'
            res[f'{key}_ms_per_batch'] = ms
            res[f'{key}_complexes_per_s'] = B * 1000.0 / ms
        ddpm.loop_engine = 'auto'

        # the parts of the native forward: the two denoiser calls and the fused terms kernel on the same shapes
        ligand, pocket = model.get_ligand_and_pocket(data)
        ligand, pocket = ddpm.normalize(ligand, pocket)
        lm, pm = ligand['mask'], pocket['mask']
        xl = torch.cat([ligand['x'], ligand['one_hot']], 1)
        xp = torch.cat([pocket['x'], pocket['one_hot']], 1)
        t = torch.full((B, 1), 0.5, device='cuda')
        res['denoiser_pair_ms'] = time_ms(lambda: (dyn(xl, xp, t, lm, pm), dyn(xl, xp, t, lm, pm)), args.batches,
                                          args.warmup)
        net = dyn(xl, xp, t, lm, pm)[0]
        gamma = ddpm.inflate_batch_array(ddpm.gamma(t), xl)
        lig_side = (xl, xl, net, net, xl, net, net)
        res['vlb_terms_call_ms'] = time_ms(lambda: ddpm._native_vlb_terms(lig_side, None, lm, pm, gamma, gamma, None),
                                             args.batches * 4, args.warmup)
    res['denoiser_share_native'] = res['denoiser_pair_ms'] / res['native_ms_per_batch']
    res['rest_ms_native'] = res['native_ms_per_batch'] - res['denoiser_pair_ms']
    res['eager_terms_ms'] = res['eager_ms_per_batch'] - res['denoiser_pair_ms']
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
