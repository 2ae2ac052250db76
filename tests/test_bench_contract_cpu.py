"""CPU: the reference arm of bench.py (`--impl reference`, the CPU port of the reference's op sequence on a bounded
sample) prints ONE JSON line with the contract's keys, on a tiny shape so that it runs in seconds.  The b200 arm needs
a GPU and is exercised on a GPU host; here only its refusal to run without one is checked."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_bench(*argv, env=None):
    e = dict(os.environ, OMP_NUM_THREADS='4')
    e.update(env or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), *argv], capture_output=True, text=True, env=e,
                          timeout=600)


def test_reference_arm_prints_contract_line():
    r = run_bench('--impl', 'reference', '--steps', '2', '--warmup', '1', '--batch', '2', '--n-lig', '4', '--n-pocket', '12',
                  '--timesteps', '20', '--cpu-sample-seconds', '0.5')
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.startswith('{')]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d['impl'] == 'reference' and d['metric'] == 'ligand_atoms_per_sec_500step_ddpm' and d['unit'] == 'ligand atoms/s'
    assert d['higher_is_better'] is True and d['steps'] == 2 and d['warmup'] == 1 and d['n_gpus'] == 1
    assert d['value'] > 0 and d['ms_per_step'] > 0
    cb = d['cpu_baseline']
    assert cb['kind'] == 'port' and cb['cores'] >= 1 and cb['value'] == d['value'] and 'denoiser calls' in cb['sample']
    assert d['e2e'] == {'value': d['value'], 'unit': d['unit'], 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}
    assert d['config']['workload'].startswith('BASELINE configs[2]')


def test_reference_arm_other_ranks_exit_quietly():
    r = run_bench('--impl', 'reference', '--steps', '1', '--warmup', '0', env={'RANK': '1', 'WORLD_SIZE': '2'})
    assert r.returncode == 0 and not [l for l in r.stdout.splitlines() if l.startswith('{')]
