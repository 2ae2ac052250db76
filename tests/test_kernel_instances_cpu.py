"""CPU: every tensor-core kernel instance compiled into the library is launched by at least one per-launch check.

The per-launch checks (tests/test_gpu_launches.py, tests/test_gpu_fast_math.py) are the sharp test of the denoiser's
kernels: whole-forward tolerances sit far above the error of one contraction, so an instance that only ever runs inside a
whole forward can lose precision unnoticed.  The library's entry symbols (``cuobjdump -symbols``, demangled with
``cu++filt``) list the instances of ``tc_node_gemm_kernel<FMT, H>`` and ``tc_edge_kernel<COORD, FMT, H, TB, DET>``;
``launch_cases.tc_instances`` says which of them one forward launches (test_gpu_launches.py checks that against the
profiler on the GPU).  The union over every per-launch parametrisation of the two GPU files must be all of them, so an
instance added without a case fails here, on a machine without a GPU.
"""
import os
import shutil
import subprocess

import pytest

import launch_cases as lc
import test_gpu_fast_math as fm
import test_gpu_launches as tl
from diffsbdd_b200 import _build

N_INSTANCES = 81      # node GEMM: 3 formats x 3 widths; edge kernels: 2 COORD x 3 formats x 3 widths x 2 TB x 2 DET


def _tool(name):
    path = shutil.which(name) or os.path.join('/usr/local/cuda/bin', name)
    assert os.path.exists(path), f'{name} (CUDA toolkit) not found'
    return path


@pytest.fixture(scope='module')
def compiled():
    out = subprocess.run([_tool('cuobjdump'), '-symbols', _build.build()], capture_output=True, text=True, check=True).stdout
    entries = [ln.split()[-1] for ln in out.splitlines() if 'STT_FUNC' in ln and 'STO_ENTRY' in ln]
    return {i for i in map(lc.parse_tc_instance, lc.demangle(entries)) if i is not None}


def per_launch_parametrisations():
    """(case, mode, det) of every per-launch test of test_gpu_launches.py and test_gpu_fast_math.py."""
    out = [(n, m, True) for n, m in tl.PARAMS] + [(n, m, False) for n, m in tl.DEFAULT_PARAMS]
    out += [('ladder_h256', m, True) for m in tl.MODES]                 # test_ladder_graph_alone_vs_batched_per_launch
    out += [(n, fm.MODE, True) for n in fm.CASES_1X] + [(n, fm.MODE, False) for n in fm.DEFAULT_CASES_1X]
    return out


def test_parse_both_spellings():
    want = ('tc_edge_kernel', True, 'F16x3', 192, True, False)
    assert lc.parse_tc_instance('void dsb::tc_edge_kernel<(bool)1, (dsb::TcFormat)1, (int)192, (bool)1, (bool)0>'
                                '(dsb::TcEdgeArgs)') == want
    assert lc.parse_tc_instance('void dsb::tc_edge_kernel<true, (dsb::TcFormat)1, 192, true, false>(dsb::TcEdgeArgs)') == want
    assert lc.parse_tc_instance('void dsb::tc_edge_kernel<true, dsb::TcFormat::F16x3, 192, true>(dsb::TcEdgeArgs)') == want
    assert lc.parse_tc_instance('void dsb::tc_node_gemm_kernel<(dsb::TcFormat)2, (int)128>(dsb::TcGemmArgs)') == \
        ('tc_node_gemm_kernel', None, 'F16x1', 128, None, None)
    assert lc.parse_tc_instance('void dsb::segment_reduce_kernel(float4*, int)') is None


def test_library_instances(compiled):
    assert len(compiled) == N_INSTANCES, sorted(map(str, compiled))
    assert {i[3] for i in compiled} == set(lc.TC_WIDTHS) and {i[2] for i in compiled} == set(lc.TC_FORMATS)


def test_every_instance_is_checked_per_launch(compiled):
    cfgs = {}
    covered = {}
    for name, mode, det in per_launch_parametrisations():
        if name not in cfgs:
            cfgs[name] = tl.case_cfg(name)
        for inst in lc.tc_instances(cfgs[name], mode, det):
            covered.setdefault(inst, []).append(f'{name} mode {mode} det {int(det)}')
    missing = sorted(compiled - set(covered), key=str)
    unknown = sorted(set(covered) - compiled, key=str)
    print(f'\n{len(compiled) - len(missing)} of {len(compiled)} tensor-core kernel instances checked per launch')
    assert not missing, 'instances no per-launch case launches:\n' + '\n'.join(map(str, missing))
    assert not unknown, 'the ledger names instances the library does not have:\n' + '\n'.join(map(str, unknown))
