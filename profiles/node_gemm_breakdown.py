"""Where the node-GEMM time goes: every `tc_node_gemm_kernel` launch of one denoiser call, timed on its own.

For each workload (bench.py's `fullatom` = configs[2], `moad`, `moad_ca`) eager forwards run after warm-up, each preceded by
bench.py's 256 MiB L2 flush, under torch.profiler (CUDA activities).  The node-GEMM launches of a forward come in a fixed
order (dsb_api.cu, dsb_dynamics_forward): per block and sub-layer the edge first layer g1 (block 0 / later sub-layers only),
the node MLP g2 (hidden layer, K = 2H) and g3 (output layer + residual, zeroes agg), then per block the merged first-layer
GEMM g4 (coordinate MLPs of this block + edge first layer of the next; receiver-side coordinate columns skipped for pocket
rows).  Each launch is labelled by its position.  Per label the script prints:
  * us per launch (median over launches and calls): the kernel's own time, from the end of the kernel before it (or its
    start, if later) to its end; and its whole profiled span, which with programmatic dependent launch also covers the
    wait for its predecessor;
  * tiles (128 x H output tiles, dead tiles skipped) and CTAs;
  * executed TFLOP/s (3 split products per MAC, padded rows of the last tile included);
  * an HBM-byte lower bound: A read once, R read once, C and Z written once;
  * the L2 weight-stream bytes: tiles x chunks x 2 (hi, lo) x H x 128 B;
and beside them the least time the data sheet allows for each (989 TFLOP/s dense FP16 / 495 TF32 and 3.35 TB/s HBM3 of a
700 W H100 SXM; data-sheet figures, not measurements).  The card name and power limit are read in the same run.
Needs a CUDA device.

    python profiles/node_gemm_breakdown.py [--workloads fullatom,moad,moad_ca] [--calls 20] [--math-mode 3xfp16] [--out f.json]
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
from diffsbdd_b200.dynamics import EGNNDynamics  # noqa: E402

TM = 128                 # rows per output tile (dsb_tc.cuh)
PEAK_TFLOPS = {'3xfp16': 989.0, '3xtf32': 495.0}
HBM_TBS = 3.35


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--id=0', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm',
                              '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip()
        return out
    except Exception:  # noqa: BLE001
        return None


def launch_plan(cfg, n, n_lig):
    """(label, K, Nn, has R, has Z, dead_rows_from, dead_cols) of every node GEMM of one forward, in launch order."""
    H = cfg.hidden_nf
    nm = 1 if cfg.reflection_equivariant else 2
    conditional = not cfg.update_pocket_coords
    plan = []
    for layer in range(cfg.n_layers):
        for sub in range(cfg.inv_sublayers):
            if not (sub == 0 and layer > 0):
                plan.append(('g1', H, 2 * H, False, False, 0, 0))
            plan.append(('g2', 2 * H, H, False, False, 0, 0))
            plan.append(('g3', H, H, True, True, 0, 0))
        plan.append(('g4', H, nm * 2 * H + 2 * H, False, False, n_lig if conditional else 0, nm * H if conditional else 0))
    return plan


def shape_counts(H, M, K, Nn, has_r, has_z, dead_from, dead_cols, f16, n_sms):
    ntn, ntm = Nn // H, (M + TM - 1) // TM
    dnt = dead_cols // H
    dmt = min((dead_from + TM - 1) // TM, ntm) if dnt > 0 else ntm
    tiles = dmt * ntn + (ntm - dmt) * (ntn - dnt)
    chunks = K // (64 if f16 else 32)
    dead_rows = max(M - dmt * TM, 0) if dnt > 0 else 0
    c_elems = M * Nn - dead_rows * dnt * H
    hbm = 4 * (M * K + (M * Nn if has_r else 0) + c_elems + (M * H if has_z else 0))
    return {'tiles': tiles, 'ctas': min(tiles, n_sms), 'chunks_per_tile': chunks,
            'exec_gflop': 6.0 * tiles * TM * H * K / 1e9, 'hbm_lb_mb': hbm / 1e6,
            'l2_weight_mb': tiles * chunks * 2 * H * 128 / 1e6}


def profile_workload(name, calls, warmup, math_mode, flush):
    a = argparse.Namespace(workload=name)
    cfg, _, _, _ = bench.workload(a)
    _, B, NL, NP, _, _, _, _ = bench.WORKLOADS[name]
    sd = syn.synthetic_state_dict(cfg, 0)
    dyn = EGNNDynamics.from_config(cfg, device='cuda')
    dyn.load_state_dict(sd)
    dyn.eval()
    dyn.math_mode = math_mode
    inp = [x.cuda() for x in syn.synthetic_denoiser_inputs(cfg, [NL] * B, [NP] * B, seed=1)]
    H, M = cfg.hidden_nf, B * (NL + NP)
    plan = launch_plan(cfg, M, B * NL)
    with torch.no_grad():
        for _ in range(warmup):
            bench.l2_flush(flush)
            dyn(*inp)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                bench.l2_flush(flush)
                dyn(*inp)
            torch.cuda.synchronize()
    # With programmatic dependent launch a kernel starts when its predecessor does and waits in griddepcontrol.wait, so
    # its profiled interval covers the predecessor's.  Its own time is end - max(start, end of every earlier kernel).
    raw = sorted(((e.start_ns(), e.start_ns() + e.duration_ns(), e.name()) for e in prof.profiler.kineto_results.events()
                  if e.device_type() == torch.autograd.DeviceType.CUDA), key=lambda t: t[0])
    kern, last_end = [], 0
    for s, e, n in raw:
        kern.append((s, max(e - max(s, last_end), 0), n, e - s))
        last_end = max(last_end, e)
    gemms = [k for k in kern if 'tc_node_gemm_kernel' in k[2]]
    if len(gemms) != calls * len(plan):
        raise SystemExit(f'{name}: {len(gemms)} node-GEMM kernels for {calls} calls, expected {len(plan)} per call')
    per_label, span = {}, {}
    for i, (_, dur, _, sp) in enumerate(gemms):
        per_label.setdefault(plan[i % len(plan)][0], []).append(dur / 1e3)
        span.setdefault(plan[i % len(plan)][0], []).append(sp / 1e3)
    classes = {'node_gemm': 'tc_node_gemm_kernel', 'edge_gcl': 'tc_edge_kernel<false', 'edge_coord': 'tc_edge_kernel<true'}
    by_class = {c: round(sum(d for _, d, n, _ in kern if key in n) / 1e6 / calls, 4) for c, key in classes.items()}
    by_class['all_dsb_kernels'] = round(sum(d for _, d, n, _ in kern if 'dsb::' in n) / 1e6 / calls, 4)
    f16 = math_mode == '3xfp16'
    rows = []
    for lab in ('g1', 'g2', 'g3', 'g4'):
        if lab not in per_label:
            continue
        p = next(x for x in plan if x[0] == lab)
        sc = shape_counts(H, M, p[1], p[2], p[3], p[4], p[5], p[6], f16, torch.cuda.get_device_properties(0).multi_processor_count)
        us = statistics.median(per_label[lab])
        rows.append({'label': lab, 'launches_per_call': len(per_label[lab]) // calls, 'M': M, 'K': p[1], 'Nn': p[2],
                     'us_median': round(us, 2), 'us_min': round(min(per_label[lab]), 2), 'us_max': round(max(per_label[lab]), 2),
                     'span_us_median': round(statistics.median(span[lab]), 2),
                     **sc, 'exec_tflops': round(sc['exec_gflop'] / us * 1e3, 1),
                     'tensor_bound_us': round(sc['exec_gflop'] / PEAK_TFLOPS[math_mode] / 1e-3, 2),
                     'hbm_bound_us': round(sc['hbm_lb_mb'] / HBM_TBS, 2),
                     'l2_weight_gbs': round(sc['l2_weight_mb'] / us * 1e3, 1)})
    node_ms = sum(r['us_median'] * r['launches_per_call'] for r in rows) / 1e3
    return {'workload': name, 'hidden_nf': H, 'M': M, 'math_mode': math_mode, 'calls': calls,
            'node_gemm_ms_per_call_from_medians': round(node_ms, 4), 'ms_per_call_by_class': by_class, 'per_label': rows}


def print_table(res):
    print(f"\n{res['workload']} (H = {res['hidden_nf']}, M = {res['M']}, {res['math_mode']}); per call: {res['ms_per_call_by_class']}")
    print('| launch | per call | us/launch (min-max) | span us | tiles | CTAs | exec TFLOP/s | tensor bound us | HBM LB MB | HBM bound us '
          '| L2 weight MB | L2 weight GB/s |')
    print('|---|---|---|---|---|---|---|---|---|---|---|---|')
    for r in res['per_label']:
        print(f"| {r['label']} | {r['launches_per_call']} | {r['us_median']} ({r['us_min']}-{r['us_max']}) | {r['span_us_median']} | {r['tiles']} | {r['ctas']} "
              f"| {r['exec_tflops']} | {r['tensor_bound_us']} | {r['hbm_lb_mb']:.1f} | {r['hbm_bound_us']} | {r['l2_weight_mb']:.1f} "
              f"| {r['l2_weight_gbs']} |")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='fullatom,moad,moad_ca')
    ap.add_argument('--calls', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--math-mode', default='3xfp16', choices=sorted(PEAK_TFLOPS))
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('node_gemm_breakdown.py needs a CUDA device')
    flush = torch.zeros(64 * 1024 * 1024, dtype=torch.float32, device='cuda')
    out = {'gpu': gpu_info(), 'torch_device': torch.cuda.get_device_name(0), 'results': []}
    print('gpu (name, power limit, SM clock, max SM clock):', out['gpu'])
    for w in args.workloads.split(','):
        res = profile_workload(w, args.calls, args.warmup, args.math_mode, flush)
        out['results'].append(res)
        print_table(res)
    print('\n(tensor / HBM bounds: data-sheet peaks of a 700 W H100 SXM, not measured; DRAM traffic is not measured)')
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
