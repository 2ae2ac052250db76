"""ctypes binding of libdiffsbdd_b200.so (include/diffsbdd_b200.h).

There is deliberately NO fallback: if the CUDA library is missing this module raises at load time, and
the product path never routes through a CPU/PyTorch re-implementation.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

from . import _build

_LIB: Optional[C.CDLL] = None

EXPORTED_SYMBOLS = (
    'dsb_param_count', 'dsb_param_name', 'dsb_dynamics_create', 'dsb_dynamics_destroy',
    'dsb_edge_capacity', 'dsb_dynamics_workspace_bytes', 'dsb_dynamics_forward', 'dsb_dynamics_edges',
    'dsb_dynamics_last_launch_count', 'dsb_set_programmatic_launch', 'dsb_dynamics_set_math_mode', 'dsb_dynamics_set_deterministic', 'dsb_dynamics_set_profiling', 'dsb_dynamics_collect_profile',
    'dsb_ddpm_ligand_update', 'dsb_ddpm_inpaint_update', 'dsb_ddpm_joint_update', 'dsb_ddpm_joint_inpaint_update', 'dsb_ddpm_noise',
    'dsb_ddpm_multistep_update', 'dsb_ddpm_multistep_inpaint_update', 'dsb_ddpm_multistep3_update',
    'dsb_ddpm_multistep3_inpaint_update',
    'dsb_ddpm_vlb_terms', 'dsb_last_error', 'dsb_version', 'dsb_dynamics_set_stop_after', 'dsb_workspace_region',
    'dsb_seeded_normal',
)

# roles and kinds of dsb_seeded_normal (DSB_RNG_* in include/diffsbdd_b200.h)
RNG_LIGAND, RNG_POCKET, RNG_JOINT_X, RNG_GRAPH = 0, 1, 2, 3
RNG_NORMAL, RNG_UNIFORM, RNG_BITS = 0, 1, 2

# workspace regions of dsb_workspace_region (DSB_WS_* in include/diffsbdd_b200.h), in enum order
WS_REGIONS = ('x_in', 'x_ping', 'x_pong', 'h', 'hT', 'agg', 'P', 'xagg', 'cent', 'deg', 'row_ptr', 'vrow_ptr', 'vmap',
              'erow', 'ecol', 'ed0', 'part', 'lig_off', 'poc_off', 'gid', 'velmean')


class DsbConfig(C.Structure):
    """``dsb_config`` of include/diffsbdd_b200.h (EGNNDynamics constructor args, dynamics.py:11-19)."""
    _fields_ = [
        ('atom_nf', C.c_int32), ('residue_nf', C.c_int32), ('n_dims', C.c_int32), ('joint_nf', C.c_int32),
        ('hidden_nf', C.c_int32), ('n_layers', C.c_int32), ('inv_sublayers', C.c_int32),
        ('attention', C.c_int32), ('tanh', C.c_int32), ('condition_time', C.c_int32),
        ('update_pocket_coords', C.c_int32), ('reflection_equivariant', C.c_int32),
        ('edge_embedding_dim', C.c_int32),
        ('norm_constant', C.c_float), ('normalization_factor', C.c_float), ('coords_range', C.c_float),
        ('edge_cutoff_ligand', C.c_float), ('edge_cutoff_pocket', C.c_float),
        ('edge_cutoff_interaction', C.c_float),
        ('aggregation_mean', C.c_int32),
        ('sin_embedding', C.c_int32),
    ]


class NativeError(RuntimeError):
    pass


def lib_path() -> str:
    return _build.LIB_PATH


def load(build_if_missing: bool = True) -> C.CDLL:
    global _LIB
    if _LIB is not None:
        return _LIB
    path = _build.LIB_PATH
    if os.environ.get('DSB_LIB_PATH'):                                  # a library built elsewhere (e.g. with other flags)
        path = os.environ['DSB_LIB_PATH']
        if not os.path.exists(path):
            raise NativeError(f'DSB_LIB_PATH={path} does not exist')
    elif not os.path.exists(path) or not _build.is_current():
        # missing, or built from other sources than the ones next to it (the .so is git-ignored and travels separately):
        # a stale library behind fixed ctypes signatures would corrupt memory silently
        if not build_if_missing:
            raise NativeError(f'{path} is missing or stale: run `python -m diffsbdd_b200._build` (needs nvcc)')
        _build.build()
    lib = C.CDLL(path)
    vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int32
    lib.dsb_last_error.restype = C.c_char_p
    lib.dsb_version.restype = C.c_char_p
    lib.dsb_param_count.argtypes = [C.POINTER(DsbConfig)]
    lib.dsb_param_count.restype = C.c_int
    lib.dsb_param_name.argtypes = [C.POINTER(DsbConfig), C.c_int, C.c_char_p, C.c_size_t]
    lib.dsb_param_name.restype = i64
    lib.dsb_dynamics_create.argtypes = [C.POINTER(DsbConfig), C.POINTER(vp), C.c_int, C.POINTER(vp)]
    lib.dsb_dynamics_create.restype = C.c_int
    lib.dsb_dynamics_destroy.argtypes = [vp]
    lib.dsb_dynamics_destroy.restype = None
    lib.dsb_edge_capacity.argtypes = [C.POINTER(i64), C.POINTER(i64), C.c_int]
    lib.dsb_edge_capacity.restype = i64
    lib.dsb_dynamics_workspace_bytes.argtypes = [vp, i64, i64, i64, i64]
    lib.dsb_dynamics_workspace_bytes.restype = C.c_size_t
    lib.dsb_dynamics_forward.argtypes = [vp, vp, vp, vp, i64, vp, vp, i64, i64, i64, i64, vp, vp, vp,
                                         C.c_size_t, vp, vp]
    lib.dsb_dynamics_forward.restype = C.c_int
    lib.dsb_dynamics_edges.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, vp, vp, vp, vp, C.c_size_t, vp]
    lib.dsb_dynamics_edges.restype = C.c_int
    lib.dsb_dynamics_last_launch_count.argtypes = [vp]
    lib.dsb_dynamics_last_launch_count.restype = C.c_int
    lib.dsb_set_programmatic_launch.argtypes = [C.c_int]
    lib.dsb_set_programmatic_launch.restype = C.c_int
    lib.dsb_dynamics_set_math_mode.argtypes = [vp, C.c_int]
    lib.dsb_dynamics_set_math_mode.restype = C.c_int
    lib.dsb_dynamics_set_deterministic.argtypes = [vp, C.c_int]
    lib.dsb_dynamics_set_deterministic.restype = C.c_int
    lib.dsb_dynamics_set_profiling.argtypes = [vp, C.c_int]
    lib.dsb_dynamics_set_profiling.restype = C.c_int
    lib.dsb_dynamics_collect_profile.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(i64), C.c_int]
    lib.dsb_dynamics_collect_profile.restype = C.c_int
    lib.dsb_ddpm_ligand_update.argtypes = [vp, vp, vp, vp, vp, vp, vp, i64, i64, i64, i32, i32, vp, vp, vp]
    lib.dsb_ddpm_ligand_update.restype = C.c_int
    lib.dsb_ddpm_inpaint_update.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i64, i64, i64, i32, i32, vp]
    lib.dsb_ddpm_inpaint_update.restype = C.c_int
    lib.dsb_ddpm_joint_update.argtypes = [vp] * 10 + [i64, i64, i64, i32, i32, vp]
    lib.dsb_ddpm_joint_update.restype = C.c_int
    lib.dsb_ddpm_joint_inpaint_update.argtypes = [vp] * 15 + [i64, i64, i64, i32, i32, vp]
    lib.dsb_ddpm_joint_inpaint_update.restype = C.c_int
    lib.dsb_ddpm_multistep_update.argtypes = [vp] * 9 + [i64, i64, i64, i32, i32, i32, vp]
    lib.dsb_ddpm_multistep_update.restype = C.c_int
    lib.dsb_ddpm_multistep_inpaint_update.argtypes = [vp] * 20 + [i64, i64, i64, i32, i32, i32, i32, vp]
    lib.dsb_ddpm_multistep_inpaint_update.restype = C.c_int
    lib.dsb_ddpm_multistep3_update.argtypes = [vp] * 11 + [i64, i64, i64, i32, i32, i32, vp]
    lib.dsb_ddpm_multistep3_update.restype = C.c_int
    lib.dsb_ddpm_multistep3_inpaint_update.argtypes = [vp] * 22 + [i64, i64, i64, i32, i32, i32, i32, vp]
    lib.dsb_ddpm_multistep3_inpaint_update.restype = C.c_int
    lib.dsb_ddpm_noise.argtypes = [vp] * 7 + [i64, i64, i64, i32, i32, vp, vp, vp]
    lib.dsb_ddpm_noise.restype = C.c_int
    lib.dsb_ddpm_vlb_terms.argtypes = [vp] * 16 + [i64, i64, i64, i32, i32, C.c_float, C.c_float, i32, vp, vp, vp]
    lib.dsb_ddpm_vlb_terms.restype = C.c_int
    lib.dsb_dynamics_set_stop_after.argtypes = [vp, C.c_int]
    lib.dsb_dynamics_set_stop_after.restype = C.c_int
    lib.dsb_workspace_region.argtypes = [C.POINTER(DsbConfig), C.c_int, i64, i64, i64, i64, C.c_int, C.POINTER(i64),
                                         C.POINTER(i64)]
    lib.dsb_workspace_region.restype = C.c_int
    lib.dsb_seeded_normal.argtypes = [vp, i64, i32, i32, vp, vp, vp, vp, i64, i64, i64, vp]
    lib.dsb_seeded_normal.restype = C.c_int
    _LIB = lib
    return lib


def workspace_regions(cfg: DsbConfig, deterministic: bool, n_atoms: int, n_residues: int, n_graphs: int,
                      edge_capacity: int):
    """{region name: (byte offset, bytes)} of the forward's workspace (dsb_workspace_region; test hook)."""
    lib = load()
    out = {}
    off, nb = C.c_int64(), C.c_int64()
    for i, name in enumerate(WS_REGIONS):
        check(lib.dsb_workspace_region(C.byref(cfg), int(bool(deterministic)), n_atoms, n_residues, n_graphs,
                                       edge_capacity, i, C.byref(off), C.byref(nb)))
        out[name] = (off.value, nb.value)
    return out


def check(code: int) -> None:
    if code != 0:
        msg = load().dsb_last_error().decode(errors='replace')
        raise NativeError(f'libdiffsbdd_b200 error {code}: {msg}')


def multistep_update(lib: C.CDLL, z, hist, eps, coef, masks, sizes, joint: int, stream, repaint=(), commit: int = 1) -> None:
    """One DPM-Solver++ step, or with ``repaint`` one RePaint round, in place on device tensors: 2M with one history, 3M with
    two (dsb_ddpm_multistep[3][_inpaint]_update).  ``z``, ``eps`` and each history, newest first: (ligand, pocket) pairs,
    None where the conditional model has no pocket part; ``repaint``: the tensors known_lig .. renoise_h_pocket of the
    RePaint entries (None where absent); ``sizes``: (n_atoms, n_residues, n_graphs, atom_nf, residue_nf)."""
    ptr = lambda x: None if x is None else x.data_ptr()
    name = 'dsb_ddpm_multistep%s%s_update' % ('3' if len(hist) == 2 else '', '_inpaint' if repaint else '')
    bufs = (*z, *(x for h in hist for x in h), *eps, *repaint, coef, *masks)
    check(getattr(lib, name)(*map(ptr, bufs), *sizes, joint, *((commit,) if repaint else ()), stream))


def param_names(cfg: DsbConfig):
    lib = load()
    n = lib.dsb_param_count(C.byref(cfg))
    if n < 0:
        check(n)
    out = []
    buf = C.create_string_buffer(256)
    for i in range(n):
        numel = lib.dsb_param_name(C.byref(cfg), i, buf, 256)
        if numel < 0:
            check(int(numel))
        out.append((buf.value.decode(), int(numel)))
    return out
