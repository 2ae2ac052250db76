"""Writes tests/golden/layout/reference_state_dict_layout.npz: the state-dict keys (in order) and shapes of the UNMODIFIED
reference ``EGNNDynamics`` for the configurations test_boundary_cpu.py checks (through oracle/ref_shim.py).

    DIFFSBDD_REFERENCE=<reference checkout> python tests/golden/make_layout_golden.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from helpers import LAYOUT_CASES  # noqa: E402
from oracle import ref_shim  # noqa: E402


def main():
    ref = ref_shim.load_reference()
    out = {}
    for name, cfg in LAYOUT_CASES.items():
        net = ref.EGNNDynamics(device='cpu', act_fn=torch.nn.SiLU(), **cfg.kwargs())
        out[name] = np.array([f'{k}:' + 'x'.join(str(d) for d in v.shape) for k, v in net.state_dict().items()])
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'layout', 'reference_state_dict_layout.npz'), **out)


if __name__ == '__main__':
    main()
