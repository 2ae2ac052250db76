"""Drop-in ``EGNNDynamics`` whose forward runs on the hand-written sm_90a kernels.

Mirrors the reference module (equivariant_diffusion/dynamics.py:10-187): same constructor signature,
same attribute names callers read (``update_pocket_coords``, ``n_dims``, ``edge_cutoff_{l,p,i}``,
``egnn``, ``device``), same ``state_dict`` keys/shapes (so reference checkpoints load unchanged), same
``forward(xh_atoms, xh_residues, t, mask_atoms, mask_residues) -> (lig_out, pocket_out)`` contract and
the same ``ValueError("NaN detected in EGNN output")`` convention.  The parameters are plain
``nn.Parameter`` leaves in a module tree that reproduces the reference key names; all arithmetic happens
in ``libdiffsbdd_b200.so`` through its C ABI (include/diffsbdd_b200.h) on the caller's CUDA stream.

Out of scope (raises loudly): autograd through the kernels (training), ``mode='gnn_dynamics'`` — not used by the
shipped sampling configs
(SURVEY.md §8(a), last row).
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import Dict, Optional, Tuple

import torch
import torch.nn as nn

from . import _native
from .config import DynamicsConfig
from .synthetic import state_dict_spec


def _parse_deterministic(value):
    if value in (True, False, 'auto'):
        return value
    if isinstance(value, str):
        v = value.strip().lower()
        if v in ('1', 'true', 'on', 'yes'):
            return True
        if v in ('0', 'false', 'off', 'no'):
            return False
        if v in ('', 'auto'):
            return 'auto'
    raise ValueError(f"deterministic must be True, False or 'auto' (DSB_DETERMINISTIC: 1, 0 or auto), got {value!r}")


class _Tree(nn.Module):
    """Parameter container that reproduces nested reference key names (e.g. ``edge_mlp.0.weight``)."""

    def child(self, name: str) -> "_Tree":
        if name not in self._modules:
            self.add_module(name, _Tree())
        return self._modules[name]

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError('parameter container: the arithmetic lives in libdiffsbdd_b200.so')


class _PlanCache:
    """Per-batch constants derived from the mask tensors (they are constant over the 501 denoiser calls
    of one sampling run): number of graphs, edge capacity, validity.  Holds strong references to the mask
    tensors so an address can never be recycled while cached."""

    def __init__(self):
        self.key = None
        self.value = None
        self.refs = None

    def get(self, mask_atoms, mask_residues, n_graphs_hint):
        key = (id(mask_atoms), id(mask_residues), mask_atoms._version, mask_residues._version,
               mask_atoms.data_ptr(), mask_residues.data_ptr(), mask_atoms.numel(), mask_residues.numel(),
               n_graphs_hint)
        if key == self.key:
            return self.value
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError('EGNNDynamics: masks changed during CUDA-graph capture; run one eager '
                               'forward with these mask tensors first')
        ma, mr = mask_atoms, mask_residues
        hi = -1
        if ma.numel():
            hi = max(hi, int(ma.max()))
        if mr.numel():
            hi = max(hi, int(mr.max()))
        B = hi + 1 if n_graphs_hint is None else n_graphs_hint
        if hi >= B or (ma.numel() and int(ma.min()) < 0) or (mr.numel() and int(mr.min()) < 0):
            raise ValueError(f'mask values must lie in [0, {B})')
        for m in (ma, mr):
            if m.numel() > 1 and not bool((m[1:] >= m[:-1]).all()):
                raise ValueError('mask_atoms/mask_residues must be non-decreasing graph ids '
                                 '(reference utils.py:146-154 builds them with repeat_interleave)')
        nl = torch.bincount(ma, minlength=B) if ma.numel() else torch.zeros(B, dtype=torch.int64, device=ma.device)
        npk = torch.bincount(mr, minlength=B) if mr.numel() else torch.zeros(B, dtype=torch.int64, device=mr.device)
        ecap = int(((nl + npk) ** 2).sum()) if B > 0 else 0
        self.key, self.value, self.refs = key, (B, ecap), (mask_atoms, mask_residues)
        return self.value


class EGNNDynamics(nn.Module):
    """reference: equivariant_diffusion/dynamics.py:10 (constructor :11-85, forward :87-167)."""

    def __init__(self, atom_nf, residue_nf, n_dims, joint_nf=16, hidden_nf=64, device='cpu',
                 act_fn=torch.nn.SiLU(), n_layers=4, attention=False, condition_time=True, tanh=False,
                 mode='egnn_dynamics', norm_constant=0, inv_sublayers=2, sin_embedding=False,
                 normalization_factor=100, aggregation_method='sum', update_pocket_coords=True,
                 edge_cutoff_ligand=None, edge_cutoff_pocket=None, edge_cutoff_interaction=None,
                 reflection_equivariant=True, edge_embedding_dim=None):
        super().__init__()
        if mode != 'egnn_dynamics':
            if mode == 'gnn_dynamics':
                # not runnable in the reference either: its forward reads self.update_pocket_coords (dynamics.py:161), which
                # only the egnn_dynamics branch of its constructor sets (dynamics.py:73) -> AttributeError on the first call
                raise NotImplementedError("mode='gnn_dynamics' is not built (unused by every shipped config and broken in the reference)")
            raise Exception("Wrong mode %s" % mode)      # dynamics.py:144-145
        if aggregation_method not in ('sum', 'mean'):
            raise ValueError("aggregation_method must be 'sum' or 'mean' (egnn_new.py:321-335)")
        if not isinstance(act_fn, nn.SiLU):
            raise NotImplementedError('only SiLU activations are built (lightning_modules.py:143)')
        self.mode = mode
        self.edge_cutoff_l = edge_cutoff_ligand
        self.edge_cutoff_p = edge_cutoff_pocket
        self.edge_cutoff_i = edge_cutoff_interaction
        self.edge_nf = 0 if edge_embedding_dim is None else edge_embedding_dim
        self.n_dims = n_dims
        self.condition_time = condition_time
        self.update_pocket_coords = update_pocket_coords
        self.node_nf = joint_nf + (1 if condition_time else 0)
        self.device = device
        self.cfg = DynamicsConfig(
            atom_nf=atom_nf, residue_nf=residue_nf, n_dims=n_dims, joint_nf=joint_nf, hidden_nf=hidden_nf,
            n_layers=n_layers, attention=bool(attention), condition_time=bool(condition_time), tanh=bool(tanh),
            mode=mode, norm_constant=norm_constant, inv_sublayers=inv_sublayers, sin_embedding=bool(sin_embedding),
            normalization_factor=normalization_factor, aggregation_method=aggregation_method,
            update_pocket_coords=bool(update_pocket_coords), edge_cutoff_ligand=edge_cutoff_ligand,
            edge_cutoff_pocket=edge_cutoff_pocket, edge_cutoff_interaction=edge_cutoff_interaction,
            reflection_equivariant=bool(reflection_equivariant), edge_embedding_dim=edge_embedding_dim)

        # ---- parameter tree with the reference's key names ------------------------------------------------
        self._param_keys = []
        for key, shape, fan_in in state_dict_spec(self.cfg):
            node = self
            parts = key.split('.')
            for part in parts[:-1]:
                if part not in node._modules:
                    node.add_module(part, _Tree())
                node = node._modules[part]
            p = nn.Parameter(torch.empty(shape, dtype=torch.float32))
            bound = 1.0 / math.sqrt(max(fan_in, 1))
            if key.endswith('coord_mlp.4.weight'):      # xavier_uniform(gain=0.001), egnn_new.py:79
                bound = 0.001 * math.sqrt(6.0 / (hidden_nf + 1))
            if key == 'edge_embedding.weight':
                nn.init.normal_(p)
            else:
                nn.init.uniform_(p, -bound, bound)
            node.register_parameter(parts[-1], p)
            self._param_keys.append(key)
        if not reflection_equivariant:                   # shared last layer (egnn_new.py:78, :85, :91)
            for k in range(n_layers):
                q = self.egnn._modules[f'e_block_{k}']._modules['gcl_equiv']
                q.child('cross_product_mlp').child('4').register_parameter(
                    'weight', q._modules['coord_mlp']._modules['4'].weight)

        self._handle: Optional[int] = None
        self._handle_sig = None
        self._handle_gen = 0               # bumped on every (re)creation of the native module: CUDA-graph caches key on it
        self._plan = _PlanCache()
        self._workspace: Optional[torch.Tensor] = None
        self._status: Optional[torch.Tensor] = None
        self.defer_status_check = False    # samplers that CUDA-graph the loop check once at the end
        # arithmetic path: bitmask 1 node GEMMs | 2 edge kernel | 4 coordinate kernel on wgmma, 8 = 3xFP16 operand split
        # instead of 3xTF32, 16 (with 8) = the single fp16 product x_hi.w_hi (fp16-grade accuracy, faster sampling);
        # 0 = fp32 FFMA kernels.  Names: 'fp32' (0), '3xtf32' (7), '3xfp16' (15), '1xfp16' (31).
        # 'auto' = '3xfp16' when hidden_nf is 128, 192 or 256 (the widths with tensor-core kernels), else 'fp32'.
        self._math_mode = os.environ.get('DSB_MATH_MODE', 'auto')
        # fixed-order receiver sums (bit-identical repeat of a call, see include/diffsbdd_b200.h): True | False | 'auto'
        # ('auto' follows torch.are_deterministic_algorithms_enabled() at call time)
        self._deterministic = _parse_deterministic(os.environ.get('DSB_DETERMINISTIC', 'auto'))
        self.to(device)

    # ---- native handle management ---------------------------------------------------------------------
    def _c_config(self) -> _native.DsbConfig:
        c = self.cfg
        neg = lambda v: -1.0 if v is None else float(v)
        return _native.DsbConfig(
            atom_nf=c.atom_nf, residue_nf=c.residue_nf, n_dims=c.n_dims, joint_nf=c.joint_nf,
            hidden_nf=c.hidden_nf, n_layers=c.n_layers, inv_sublayers=c.inv_sublayers,
            attention=int(c.attention), tanh=int(c.tanh), condition_time=int(c.condition_time),
            update_pocket_coords=int(c.update_pocket_coords),
            reflection_equivariant=int(c.reflection_equivariant),
            edge_embedding_dim=int(c.edge_embedding_dim or 0),
            norm_constant=float(c.norm_constant), normalization_factor=float(c.normalization_factor),
            coords_range=15.0,   # the blocks receive the undivided value (egnn_new.py:197 vs :218)
            edge_cutoff_ligand=neg(c.edge_cutoff_ligand), edge_cutoff_pocket=neg(c.edge_cutoff_pocket),
            edge_cutoff_interaction=neg(c.edge_cutoff_interaction),
            aggregation_mean=int(c.aggregation_method == 'mean'), sin_embedding=int(c.sin_embedding))

    @property
    def math_mode(self) -> int:
        m = self._math_mode
        if m in ('auto', None):
            # sin_embedding (unused by every shipped config) is built in the fp32 FFMA kernels only
            return 15 if self.cfg.hidden_nf in (128, 192, 256) and not self.cfg.sin_embedding else 0
        if m == 'fp32':
            return 0
        if m == '3xtf32':
            return 7
        if m == '3xfp16':
            return 15
        if m == '1xfp16':
            return 31
        return int(m)

    @math_mode.setter
    def math_mode(self, value):
        self._math_mode = value
        if self._handle is not None:
            _native.check(_native.load().dsb_dynamics_set_math_mode(C.c_void_p(self._handle), self.math_mode))

    @property
    def deterministic(self):
        """Deterministic mode setting: ``'auto'`` (default: follows ``torch.are_deterministic_algorithms_enabled()`` at
        call time), ``True`` or ``False``.  Initial value from the environment variable ``DSB_DETERMINISTIC``
        (``1``/``0``/``auto``).  When active, one forward gives bit-identical outputs for bit-identical inputs, weights and
        math mode (same GPU model and library build), and the DDPM wrappers' per-graph sums avoid unordered atomics."""
        return self._deterministic

    @deterministic.setter
    def deterministic(self, value):
        self._deterministic = _parse_deterministic(value)

    @property
    def deterministic_active(self) -> bool:
        """The effective mode of the next forward (``'auto'`` resolved against torch's deterministic switch)."""
        d = self._deterministic
        return torch.are_deterministic_algorithms_enabled() if d == 'auto' else bool(d)

    def _params_by_key(self) -> Dict[str, torch.Tensor]:
        return dict(self.named_parameters(remove_duplicate=False))

    def _release(self):
        if self._handle is not None:
            _native.load().dsb_dynamics_destroy(C.c_void_p(self._handle))
            self._handle = None
            self._handle_sig = None

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def refresh_weights(self):
        """Re-pack the weights for the kernels (automatic when a parameter's storage/version changes)."""
        self._release()

    def _ensure_handle(self, device: torch.device):
        params = self._params_by_key()
        sig = (device,) + tuple((params[k].data_ptr(), params[k]._version) for k in self._param_keys)
        if self._handle is not None and sig == self._handle_sig:
            return
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError('EGNNDynamics: weights changed during CUDA-graph capture')
        self._release()
        lib = _native.load()
        ccfg = self._c_config()
        names = _native.param_names(ccfg)
        keep, ptrs = [], (C.c_void_p * len(names))()
        for i, (name, numel) in enumerate(names):
            p = params[name]
            if p.device != device:
                raise RuntimeError(f'parameter {name} is on {p.device}, inputs on {device}')
            t = p.detach().to(torch.float32).contiguous()
            if t.numel() != numel:
                raise RuntimeError(f'parameter {name}: expected {numel} elements, got {t.numel()}')
            keep.append(t)
            ptrs[i] = t.data_ptr()
        out = C.c_void_p()
        with torch.cuda.device(device):
            torch.cuda.current_stream().synchronize()
            _native.check(lib.dsb_dynamics_create(C.byref(ccfg), ptrs, len(names), C.byref(out)))
        self._handle, self._handle_sig = out.value, sig
        self._handle_gen += 1
        _native.check(lib.dsb_dynamics_set_math_mode(C.c_void_p(self._handle), self.math_mode))

    def capture_signature(self):
        """Everything a captured CUDA graph of ``forward`` bakes in besides the batch layout: the native module (packed
        weight blob), the kernel selection and the scratch/status buffers.  Samplers that replay captured graphs compare
        this before every run and re-capture on a mismatch."""
        ws = self._workspace.data_ptr() if self._workspace is not None else 0
        stt = self._status.data_ptr() if self._status is not None else 0
        pdl = int(_native.load().dsb_set_programmatic_launch(-1))
        return (self._handle_gen, self._handle, self.math_mode, ws, stt, pdl, self.deterministic_active)

    def _scratch(self, device, n_atoms, n_res, n_graphs, ecap) -> torch.Tensor:
        lib = _native.load()
        need = int(lib.dsb_dynamics_workspace_bytes(C.c_void_p(self._handle), n_atoms, n_res, n_graphs, ecap))
        if need == 0:
            _native.check(-1)
        ws = self._workspace
        if ws is None or ws.device != device or ws.numel() < need:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError('EGNNDynamics: workspace would grow during CUDA-graph capture; run one '
                                   'eager forward with these shapes first')
            ws = torch.empty(need, dtype=torch.uint8, device=device)
            self._workspace = ws
        if self._status is None or self._status.device != device:
            self._status = torch.zeros(4, dtype=torch.int32, device=device)
        return ws

    def check_status(self):
        """Turns the sticky device flags into the reference's exceptions (dynamics.py:155-159)."""
        if self._status is None:
            return
        flags = self._status.tolist()
        if flags[0] or flags[2]:
            self._status.zero_()
        if flags[2]:
            raise RuntimeError('edge list overflowed edge_capacity (internal error)')
        if flags[0]:
            # dynamics.py:155-159.  In the 3xFP16 arithmetic an activation beyond the fp16 range (|x| > 65504) also ends
            # here (inf -> NaN); the range-robust alternative is named in the message.
            hint = " (if the inputs are finite: an activation may have left the fp16 range of math_mode='3xfp16' - " \
                   "set math_mode='3xtf32')" if (self.math_mode & 8) else ''
            raise ValueError('NaN detected in EGNN output' + hint)

    @property
    def last_num_edges(self) -> int:
        return int(self._status[1]) if self._status is not None else 0

    @property
    def launches_per_forward(self) -> int:
        if self._handle is None:
            return 0
        return int(_native.load().dsb_dynamics_last_launch_count(C.c_void_p(self._handle)))

    PROFILE_CLASSES = ('setup', 'node_gemm', 'memset', 'edge_gcl', 'edge_coord', 'coord_finish', 'post')

    def set_profiling(self, enabled: bool):
        """Per-kernel-class CUDA-event timing of eager (non-captured) forwards; see include/diffsbdd_b200.h."""
        if self._handle is None:
            raise RuntimeError('run one forward first (the native module is created lazily)')
        _native.check(_native.load().dsb_dynamics_set_profiling(C.c_void_p(self._handle), int(bool(enabled))))

    def collect_profile(self, reset: bool = True):
        ms = (C.c_double * 7)()
        cnt = (C.c_int64 * 7)()
        _native.check(_native.load().dsb_dynamics_collect_profile(C.c_void_p(self._handle), ms, cnt, int(reset)))
        return {k: {'ms': ms[i], 'intervals': cnt[i]} for i, k in enumerate(self.PROFILE_CLASSES)}

    # ---- the hot path ----------------------------------------------------------------------------------
    def _prepare(self, xh_atoms, xh_residues, mask_atoms, mask_residues, n_graphs_hint):
        device = xh_atoms.device
        if device.type != 'cuda':
            raise RuntimeError('diffsbdd_b200.EGNNDynamics runs only on CUDA tensors (no CPU fallback); '
                               f'got {device}')
        for name, tns in (('xh_residues', xh_residues), ('mask_atoms', mask_atoms), ('mask_residues', mask_residues)):
            if tns.device != device:
                raise RuntimeError(f'{name} is on {tns.device}, xh_atoms on {device}')
        A, R = self.cfg.atom_nf, self.cfg.residue_nf
        if xh_atoms.dim() != 2 or xh_atoms.shape[1] != self.n_dims + A:
            raise RuntimeError(f'xh_atoms must be [N_L, {self.n_dims + A}], got {tuple(xh_atoms.shape)}')
        if xh_residues.dim() != 2 or xh_residues.shape[1] != self.n_dims + R:
            raise RuntimeError(f'xh_residues must be [N_P, {self.n_dims + R}], got {tuple(xh_residues.shape)}')
        if mask_atoms.shape != (xh_atoms.shape[0],) or mask_residues.shape != (xh_residues.shape[0],):
            raise RuntimeError('mask shapes do not match the node tensors')
        if mask_atoms.dtype != torch.int64 or mask_residues.dtype != torch.int64:
            raise RuntimeError('masks must be int64 (reference constants.py:9)')
        self._ensure_handle(device)
        rc = _native.load().dsb_dynamics_set_deterministic(C.c_void_p(self._handle), int(self.deterministic_active))
        if rc < 0:
            _native.check(rc)
        n_graphs, ecap = self._plan.get(mask_atoms, mask_residues, n_graphs_hint)
        ws = self._scratch(device, xh_atoms.shape[0], xh_residues.shape[0], n_graphs, ecap)
        return device, n_graphs, ecap, ws

    def forward(self, xh_atoms, xh_residues, t, mask_atoms, mask_residues):
        if torch.is_grad_enabled() and (self.training or xh_atoms.requires_grad or xh_residues.requires_grad):
            raise NotImplementedError('diffsbdd_b200.EGNNDynamics is inference-only: call under torch.no_grad() '
                                      'in eval mode (training/autograd is out of scope, SURVEY.md §8)')
        t_flat = t.reshape(-1)
        hint = int(t_flat.numel()) if (self.condition_time and t_flat.numel() > 1) else None
        device, n_graphs, ecap, ws = self._prepare(xh_atoms, xh_residues, mask_atoms, mask_residues, hint)
        xa = xh_atoms.detach().to(torch.float32).contiguous()
        xr = xh_residues.detach().to(torch.float32).contiguous()
        tt = t_flat.detach().to(device=device, dtype=torch.float32).contiguous()
        ma, mr = mask_atoms.contiguous(), mask_residues.contiguous()
        out_a = torch.empty_like(xa)
        out_r = torch.empty_like(xr)
        lib = _native.load()
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream().cuda_stream
            _native.check(lib.dsb_dynamics_forward(
                C.c_void_p(self._handle), xa.data_ptr(), xr.data_ptr(), tt.data_ptr(), tt.numel(),
                ma.data_ptr(), mr.data_ptr(), xa.shape[0], xr.shape[0], n_graphs, ecap,
                out_a.data_ptr(), out_r.data_ptr(), ws.data_ptr(), ws.numel(),
                self._status.data_ptr(), C.c_void_p(stream)))
        if not self.defer_status_check:
            self.check_status()
        return out_a, out_r

    @torch.no_grad()
    def get_edges(self, batch_mask_ligand, batch_mask_pocket, x_ligand, x_pocket):
        """reference dynamics.py:169-187 -> int64 [2, E], sorted by (row, col)."""
        A, R = self.cfg.atom_nf, self.cfg.residue_nf
        xa = torch.zeros((x_ligand.shape[0], 3 + A), dtype=torch.float32, device=x_ligand.device)
        xr = torch.zeros((x_pocket.shape[0], 3 + R), dtype=torch.float32, device=x_pocket.device)
        xa[:, :3] = x_ligand
        xr[:, :3] = x_pocket
        device, n_graphs, ecap, ws = self._prepare(xa, xr, batch_mask_ligand, batch_mask_pocket, None)
        rows = torch.empty(ecap + 1, dtype=torch.int32, device=device)
        cols = torch.empty(ecap + 1, dtype=torch.int32, device=device)
        n_e = torch.zeros(1, dtype=torch.int32, device=device)
        lib = _native.load()
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream().cuda_stream
            _native.check(lib.dsb_dynamics_edges(
                C.c_void_p(self._handle), xa.data_ptr(), xr.data_ptr(),
                batch_mask_ligand.contiguous().data_ptr(), batch_mask_pocket.contiguous().data_ptr(),
                xa.shape[0], xr.shape[0], n_graphs, ecap, rows.data_ptr(), cols.data_ptr(), n_e.data_ptr(),
                ws.data_ptr(), ws.numel(), C.c_void_p(stream)))
        E = int(n_e)
        return torch.stack((rows[:E].long(), cols[:E].long()), dim=0)

    # ---- conveniences ------------------------------------------------------------------------------------
    @classmethod
    def from_config(cls, cfg: DynamicsConfig, device='cpu') -> "EGNNDynamics":
        return cls(device=device, act_fn=nn.SiLU(), **cfg.kwargs())
