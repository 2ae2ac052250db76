"""Float64 restatement of every floating-point launch of the native forward, one launch at a time.

``dsb_dynamics_set_stop_after`` stops the forward after any of its operations and ``dsb_workspace_region`` says where each
buffer lives in the workspace, so a test can read the state a launch starts from and the state it leaves.  This module
restates what each launch computes, from that state and from the fp32 state-dict weights (never from the packed weight
images), following the factorised algebra of DESIGN.md §2:

* ``prep``: encoders (Linear-SiLU-Linear), time channel and embedding          -> h
* ``g1``: the edge MLP's first layer, receiver | sender blocks                  -> P[:, nq:nq + 2H]
* ``gcl``: edge MLP, attention gate, raw receiver sums (after the segment reduce in deterministic mode) -> agg
* ``g2``: SiLU([h | agg / div] W3 + b3), div = normalization_factor or the receiver degree ('mean')      -> hT
* ``g3``: h + hT W4 + b4, and agg re-armed to 0                                -> h, agg
* ``g4``: coord | cross receiver, coord | cross sender, next edge MLP receiver | sender                  -> P
* ``coord``: coordinate / cross-product MLPs, tanh, coords_range, raw receiver sums of the moving nodes  -> xagg
* ``finish``: x + xagg / div for the moving nodes, xagg re-armed, per-graph centroid; ``centroid``: the centroid alone
* ``post``: velocity (joint: per-graph mean removed), folded embedding_out + decoders                   -> outputs

Each restatement returns, per output, the value and (in float64) a rigorous worst-case bound of the error of an fp32
implementation that follows the kernel's arithmetic (see ``Arith``).  ``emulate`` chains the restatements in fp32 into a
whole forward, which the CPU tests hold to the float64 oracle: that pins the restatements to the reference algebra.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from diffsbdd_b200 import synthetic as syn
from diffsbdd_b200.config import DynamicsConfig, FULLATOM_COND

U = 2.0 ** -24                     # unit roundoff of fp32


def gam(n):
    return n * U / (1 - n * U)


TC_WIDTHS = (128, 192, 256)


def effective_mode(cfg, mode):
    return mode if cfg.hidden_nf in TC_WIDTHS and not cfg.sin_embedding else 0


def nm_of(cfg):
    return 1 if cfg.reflection_equivariant else 2


# ---- the forward's operation order (dsb_api.cu, dsb_dynamics_forward) -----------------------------------------------
@dataclass
class Op:
    kind: str
    layer: int = -1
    sub: int = -1
    x_old: str = ''
    x_new: str = ''


def op_sequence(cfg, det: bool) -> List[Op]:
    """Every operation (kernel launch or memset) dsb_dynamics_forward enqueues, in order."""
    ops = [Op('plan'), Op('prep'), Op('edges_count'), Op('scan'), Op('edges_fill')]
    if nm_of(cfg) == 2:
        ops.append(Op('centroid', x_old='x_in'))
    ops += [Op('memset_agg'), Op('memset_xagg')]
    xcur = 'x_in'
    for l in range(cfg.n_layers):
        for s in range(cfg.inv_sublayers):
            if not (s == 0 and l > 0):
                ops.append(Op('g1', l, s))
            ops.append(Op('gcl', l, s, x_old=xcur))
            if det:
                ops.append(Op('segred_agg', l, s))
            ops += [Op('g2', l, s), Op('g3', l, s)]
        ops.append(Op('g4', l))
        ops.append(Op('coord', l, x_old=xcur))
        if det:
            ops.append(Op('segred_xagg', l))
        xnext = 'x_ping' if l % 2 == 0 else 'x_pong'
        ops.append(Op('finish', l, x_old=xcur, x_new=xnext))
        xcur = xnext
    if cfg.update_pocket_coords:
        ops.append(Op('velmean', x_old=xcur))
    ops.append(Op('post', x_old=xcur))
    return ops


# launch groups checked as one unit: (first op, ops it spans)
GROUPS = {'gcl': ('segred_agg',), 'coord': ('segred_xagg',), 'velmean': ('post',)}
CHECKED = ('prep', 'g1', 'gcl', 'g2', 'g3', 'g4', 'coord', 'finish', 'centroid', 'velmean', 'post')


def launch_units(cfg, det):
    """[(first op index, one past the last op index, Op)] of the checked launches (a unit spans its segment reduce in
    deterministic mode, and velmean + post in joint mode)."""
    ops = op_sequence(cfg, det)
    out, i = [], 0
    while i < len(ops):
        j = i + 1
        while j < len(ops) and ops[j].kind in GROUPS.get(ops[i].kind, ()):
            j += 1
        if ops[i].kind in CHECKED:
            out.append((i, j, ops[i]))
        i = j
    return out


# ---- state -------------------------------------------------------------------------------------------------------
@dataclass
class Dims:
    NL: int
    NP: int
    B: int
    E: int = 0

    @property
    def N(self):
        return self.NL + self.NP


def read_state(ws: torch.Tensor, regions, cfg, dm: Dims) -> Dict[str, torch.Tensor]:
    """Views of the workspace buffers a restatement reads, in logical shapes (no copy)."""
    H, N, B = cfg.hidden_nf, dm.N, dm.B

    def v(name, dtype, shape):
        off = regions[name][0]
        n = math.prod(shape) * torch.tensor([], dtype=dtype).element_size()
        assert n <= regions[name][1], (name, n, regions[name])
        return ws[off:off + n].view(dtype).view(shape)

    S = {k: v(k, torch.float32, (N, 4)) for k in ('x_in', 'x_ping', 'x_pong', 'xagg')}
    S.update(h=v('h', torch.float32, (N, H)), hT=v('hT', torch.float32, (N, H)), agg=v('agg', torch.float32, (N, H)),
             P=v('P', torch.float32, (N, (2 * nm_of(cfg) + 2) * H)),       # leading dimension (2 nm + 2) H
             cent=v('cent', torch.float32, (B, 4)), velmean=v('velmean', torch.float32, (B, 4)),
             deg=v('deg', torch.int32, (N,)), row_ptr=v('row_ptr', torch.int32, (N + 1,)),
             gid=v('gid', torch.int32, (N,)))
    E = int(S['row_ptr'][N])
    S.update(erow=v('erow', torch.int32, (E,)), ecol=v('ecol', torch.int32, (E,)), ed0=v('ed0', torch.float32, (E,)))
    return S


# ---- arithmetic model ---------------------------------------------------------------------------------------------
class Arith:
    """Worst-case error of one contraction y = sum_k a_k w_k (+ b) as the kernel evaluates it, in float64.

    M = sum_k |a_k| |w_k| (+ |b|).  fp32 FFMA (any summation order): gamma_{K+2} M.  3-product split on wgmma (x.w ~=
    x_lo w_hi + x_hi w_lo + x_hi w_hi):
    * operand split: |a_lo w_lo| <= 2^-22 |a||w| is dropped; the low parts are rounded (fp16, 2^-22 relative) or truncated
      by the MMA (tf32, 2^-21 relative each), so the split costs at most 5 * 2^-22 |a||w| per product: 2^-19 M is used;
    * 3xFP16 adds absolute floors: an activation below fp16's normal range has hi and lo parts on the 2^-24 subnormal grid
      (2^-25 |w| per product), and a weight residual below the normal range of the scaled image costs 2^-25 / scale |a|,
      with 1 / scale <= max|W| / 4096 (the image scale puts max|W| into [4096, 8192));
    * accumulation: no round-to-nearest is assumed.  One wgmma adds kg products (kg = 8 tf32, 16 fp16) to the fp32
      accumulator; if it aligns them to the largest exponent and truncates, each of the kg + 1 addends loses < 1 ulp of
      the largest magnitude, i.e. <= (kg + 1) 2u M' per instruction, with M' <= 1.01 M bounding every partial sum and
      split product.  3 K / kg instructions: 6 (K / kg)(kg + 1) u * 1.01 M;
    * epilogue (x * inv_scale + b, one fma): one rounding of the result."""

    def __init__(self, tc: bool, f16: bool):
        self.tc, self.f16 = tc, f16

    def coef(self, K):
        if not self.tc:
            return gam(K + 2)
        kg = 16 if self.f16 else 8
        return 2.0 ** -19 + 6 * math.ceil(K / kg) * (kg + 1) * U * 1.01 + 2 * U

    def floor(self, a_abs, W_abs, wmax):
        if not (self.tc and self.f16):
            return 0.0
        return 2.0 ** -25 * (W_abs.sum(1)[None, :] + a_abs.sum(1, keepdim=True) * (wmax / 4096.0))


def silu_err(x, y):
    """Bound of |silu_kernel(x) - silu(x)| for the kernels' ex2.approx / rcp.approx forms (also the shared-reciprocal
    silu4q with its exponent clamp at 31 (x < -21.5) and the ftz underflow): relative 2^-18 + |x| 2^-21 (the exponent
    argument's rounding), and the whole value where the clamp or underflow applies."""
    return y.abs() * (2.0 ** -18 + x.abs() * 2.0 ** -21) + torch.where(x < -21.0, y.abs(), torch.zeros_like(y))


def sigmoid_err(x, y):
    return y.abs() * (2.0 ** -18 + x.abs() * 2.0 ** -21) + 1e-30


def silu_b(x, ex):
    """SiLU of a value with error bound ex: value and bound (|SiLU'| <= 1.1)."""
    y = F.silu(x)
    return y, 1.1 * ex + silu_err(x, y)


def linear_b(a, ea, W, b, ar: Arith, wmax=None):
    """a [R, K] @ W[N, K]^T + b with error bound (ea: bound of a's own error)."""
    y = a @ W.T
    if b is not None:
        y = y + b
    if ea is None:
        return y, None
    Wa, aa = W.abs(), a.abs()
    M = aa @ Wa.T + (b.abs() if b is not None else 0.0)
    e = ar.coef(a.shape[1]) * M + ar.floor(aa, Wa, float(Wa.max()) if wmax is None else wmax)
    if isinstance(ea, torch.Tensor):
        e = e + ea @ Wa.T
    return y, e


# ---- restatements -----------------------------------------------------------------------------------------------
class Restater:
    """Restatements of the launches of one configuration and math mode.  ``dtype`` float64 gives the reference value and
    the bound; float32 gives the 'plain fp32 evaluation' the statistical criterion compares against (no bound)."""

    def __init__(self, cfg: DynamicsConfig, sd, inputs, mode: int, dtype=torch.float64, device='cpu'):
        self.cfg, self.dtype, self.device = cfg, dtype, device
        self.sd = {k: v.detach().to(device, dtype) for k, v in sd.items()}
        self.inp = [x.to(device) for x in inputs]
        self.bound = dtype == torch.float64
        mm = effective_mode(cfg, mode)
        f16 = bool(mm & 8)
        self.ar_node, self.ar_gcl, self.ar_coord = Arith(bool(mm & 1), f16), Arith(bool(mm & 2), f16), Arith(bool(mm & 4), f16)
        self.ar_ffma = Arith(False, False)
        NL, NP = len(inputs[3]), len(inputs[4])
        B = max(int(inputs[3].max()) + 1 if NL else 0, int(inputs[4].max()) + 1 if NP else 0)
        if cfg.condition_time and inputs[2].numel() > 1:
            B = inputs[2].numel()
        self.dm = Dims(NL, NP, B)
        self.n_coord_rows = self.dm.N if cfg.update_pocket_coords else NL
        self.H, self.nm = cfg.hidden_nf, nm_of(cfg)
        self.nq = self.nm * 2 * self.H

    def t(self, x):
        return x.to(self.device, self.dtype)

    def _e(self, v):
        return torch.zeros_like(v) if self.bound else None

    # prep: h = embedding([encoder(h_in) | t]) with the encoder's second Linear and the embedding folded (rounded once)
    def prep(self, S):
        sd, cfg, dm = self.sd, self.cfg, self.dm
        xa, xr, t, ma, mr = self.inp
        J = cfg.joint_nf
        embW, embB = sd['egnn.embedding.weight'], sd['egnn.embedding.bias']
        hs, es = [], []
        for pre, xh, mask in (('atom_encoder', xa, ma), ('residue_encoder', xr, mr)):
            f = self.t(xh[:, 3:])
            z, ez = linear_b(f, self._e(f), sd[pre + '.0.weight'], sd[pre + '.0.bias'], self.ar_ffma)
            hid, ehid = silu_b(z, ez) if self.bound else (F.silu(z), None)
            Wf = embW[:, :J] @ sd[pre + '.2.weight']                  # folded pair [H, F2]
            bf = embB + embW[:, :J] @ sd[pre + '.2.bias']
            cols, Ws = [hid], [Wf]
            if cfg.condition_time:
                tt = self.t(t.reshape(-1))
                tcol = (tt[0].expand(len(mask)) if tt.numel() == 1 else tt[mask]).reshape(-1, 1)
                cols.append(tcol)
                Ws.append(embW[:, J:J + 1])
            a, W = torch.cat(cols, 1), torch.cat(Ws, 1)
            ea = torch.cat([ehid, torch.zeros_like(cols[-1])], 1) if (self.bound and len(cols) == 2) else ehid
            y, e = linear_b(a, ea, W, bf, self.ar_ffma)
            if self.bound:      # the folded weights and bias are rounded to fp32 once
                e = e + U * (a.abs() @ W.abs().T + bf.abs())
            hs.append(y)
            es.append(e)
        return {'h': (torch.cat(hs, 0), torch.cat(es, 0) if self.bound else None)}

    def _node_gemm(self, a, ea, W, b, wmax=None):
        return linear_b(a, ea, W, b, self.ar_node, wmax)

    def g1(self, S, l, s):
        H, sd = self.H, self.sd
        W = sd[f'egnn.e_block_{l}.gcl_{s}.edge_mlp.0.weight']
        h = self.t(S['h'])
        Wab = torch.cat([W[:, :H], W[:, H:2 * H]], 0)
        b = torch.cat([sd[f'egnn.e_block_{l}.gcl_{s}.edge_mlp.0.bias'], torch.zeros_like(W[:, 0])])
        y, e = self._node_gemm(h, self._e(h), Wab, b)
        return {'P': (y, e, slice(self.nq, self.nq + 2 * H))}

    def g2(self, S, l, s):
        cfg, sd = self.cfg, self.sd
        g = f'egnn.e_block_{l}.gcl_{s}'
        h, agg = self.t(S['h']), self.t(S['agg'])
        if cfg.aggregation_method == 'mean':
            div = self.t(S['deg']).clamp(min=1)[:, None]
        else:
            div = cfg.normalization_factor
        a2 = agg / div
        a = torch.cat([h, a2], 1)
        ea = torch.cat([torch.zeros_like(h), U * a2.abs()], 1) if self.bound else None
        y, e = self._node_gemm(a, ea, sd[g + '.node_mlp.0.weight'], sd[g + '.node_mlp.0.bias'])
        if not self.bound:
            return {'hT': (F.silu(y), None)}
        y2, e2 = silu_b(y, e + U * y.abs())
        return {'hT': (y2, e2)}

    def g3(self, S, l, s):
        sd = self.sd
        g = f'egnn.e_block_{l}.gcl_{s}'
        h, hT = self.t(S['h']), self.t(S['hT'])
        y, e = self._node_gemm(hT, self._e(hT), sd[g + '.node_mlp.2.weight'], sd[g + '.node_mlp.2.bias'])
        out = h + y
        if self.bound:
            e = e + U * (out.abs() + y.abs())
        return {'h': (out, e), 'agg': (torch.zeros_like(out), None)}

    def g4(self, S, l):
        cfg, sd, H, nm = self.cfg, self.sd, self.H, self.nm
        q = f'egnn.e_block_{l}.gcl_equiv'
        names = ['coord_mlp', 'cross_product_mlp'][:nm]
        Ws = [sd[f'{q}.{m}.0.weight'] for m in names]
        blocks = [W[:, :H] for W in Ws] + [W[:, H:2 * H] for W in Ws]
        bias = [sd[f'{q}.{m}.0.bias'] for m in names] + [torch.zeros_like(Ws[0][:, 0])] * nm
        if l + 1 < cfg.n_layers:
            Wn = sd[f'egnn.e_block_{l + 1}.gcl_0.edge_mlp.0.weight']
            blocks += [Wn[:, :H], Wn[:, H:2 * H]]
            bias += [sd[f'egnn.e_block_{l + 1}.gcl_0.edge_mlp.0.bias'], torch.zeros_like(Wn[:, 0])]
        W, b = torch.cat(blocks, 0), torch.cat(bias)
        h = self.t(S['h'])
        y, e = self._node_gemm(h, self._e(h), W, b)
        return {'P': (y, e, slice(0, W.shape[0]))}

    # ---- edge kernels
    def _edges(self, S, x_old):
        er, ec = S['erow'].to(self.device).long(), S['ecol'].to(self.device).long()
        x = self.t(S[x_old][:, :3])
        return er, ec, x

    def _first_layer(self, S, W1, b1, P_recv, P_send, er, ec, x, d0):
        """u = P[recv] + P[send] + d^2 w_r + d0^2 w_r0 (+ W1e emb[type]) per edge, and its bound: the kernel adds the four
        terms in fp32 (4 roundings), d^2 from fp32 coordinates (<= 5u d^2), the type table rounded by an fp32 dot product."""
        cfg, H, NL = self.cfg, self.H, self.dm.NL
        diff = x[er] - x[ec]
        d2 = (diff * diff).sum(1, keepdim=True)
        wr, wr0 = W1[:, 2 * H], W1[:, 2 * H + 1]
        pr, ps = self.t(P_recv[er]), self.t(P_send[ec])
        u = pr + ps + d2 * wr + d0[:, None] * wr0
        tb_abs = 0.0
        if cfg.edge_embedding_dim:
            emb = self.sd['edge_embedding.weight']
            W1e = W1[:, 2 * H + 2:]
            ty = torch.zeros_like(er)
            ty[(er < NL) & (ec < NL)] = 1
            ty[(er >= NL) & (ec >= NL)] = 2
            tb = (emb @ W1e.T)[ty]
            u = u + tb
            tb_abs = (emb.abs() @ W1e.abs().T)[ty]
        if not self.bound:
            return u, None, d2
        ab = pr.abs() + ps.abs() + (d2 * wr).abs() + (d0[:, None] * wr0).abs()
        eu = gam(5) * (ab + (tb_abs if cfg.edge_embedding_dim else 0.0)) + 5 * U * d2 * wr.abs()
        if cfg.edge_embedding_dim:
            eu = eu + gam(cfg.edge_embedding_dim + 1) * tb_abs
        return u, eu, d2

    def _mlp2(self, u, eu, W2, b2, ar):
        """m = SiLU(SiLU(u) W2^T + b2) with bound."""
        if not self.bound:
            return F.silu(F.silu(u) @ W2.T + b2), None
        a, ea = silu_b(u, eu)
        y, e = linear_b(a, ea, W2, b2, ar)
        return silu_b(y, e)

    def gcl(self, S, l, s, x_old, chunk=1 << 15):
        cfg, sd, H = self.cfg, self.sd, self.H
        g = f'egnn.e_block_{l}.gcl_{s}'
        W1, W2, b2 = sd[g + '.edge_mlp.0.weight'], sd[g + '.edge_mlp.2.weight'], sd[g + '.edge_mlp.2.bias']
        er, ec, x = self._edges(S, x_old)
        d0 = self.t(S['ed0'])
        P = S['P']
        N = self.dm.N
        agg = torch.zeros((N, H), dtype=self.dtype, device=self.device)
        eagg = torch.zeros_like(agg) if self.bound else None
        sabs = torch.zeros_like(agg) if self.bound else None
        for c0 in range(0, len(er), chunk):
            sl = slice(c0, c0 + chunk)
            u, eu, _ = self._first_layer(S, W1, None, P[:, self.nq:self.nq + H], P[:, self.nq + H:self.nq + 2 * H],
                                         er[sl], ec[sl], x, d0[sl])
            m, em = self._mlp2(u, eu, W2, b2, self.ar_gcl)
            if cfg.attention:
                wa, ba = sd[g + '.att_mlp.0.weight'][0], sd[g + '.att_mlp.0.bias']
                sc = m @ wa + ba
                gate = torch.sigmoid(sc)
                if self.bound:
                    es = em @ wa.abs() + gam(H + 2) * (m.abs() @ wa.abs() + ba.abs())
                    eg = 0.25 * es + sigmoid_err(sc, gate)
                    em = gate.abs()[:, None] * em + m.abs() * eg[:, None] + U * (gate[:, None] * m).abs()
                m = m * gate[:, None]
            agg.index_add_(0, er[sl], m)
            if self.bound:
                eagg.index_add_(0, er[sl], em)
                sabs.index_add_(0, er[sl], m.abs())
        if self.bound:
            deg = torch.bincount(er, minlength=N).to(self.dtype)[:, None]
            eagg = eagg + (deg + 2) * U / (1 - (deg + 2) * U) * sabs
        return {'agg': (agg, eagg)}

    def coord(self, S, l, x_old, chunk=1 << 15):
        cfg, sd, H, nm = self.cfg, self.sd, self.H, self.nm
        q = f'egnn.e_block_{l}.gcl_equiv'
        er, ec, x = self._edges(S, x_old)
        keep = er < self.n_coord_rows
        er, ec = er[keep], ec[keep]
        d0 = self.t(S['ed0'])[keep]
        P = S['P']
        nc, rng = float(cfg.norm_constant), 15.0      # the blocks receive the undivided coords_range (egnn_new.py:218)
        w3 = sd[q + '.coord_mlp.4.weight'][0]
        N = self.dm.N
        xagg = torch.zeros((N, 3), dtype=self.dtype, device=self.device)
        ex = torch.zeros_like(xagg) if self.bound else None
        sabs = torch.zeros_like(xagg) if self.bound else None
        cent = self.t(S['cent'][:, :3])
        gid = S['gid'].to(self.device).long()
        for c0 in range(0, len(er), chunk):
            sl = slice(c0, c0 + chunk)
            r, c = er[sl], ec[sl]
            trans = torch.zeros((len(r), 3), dtype=self.dtype, device=self.device)
            et = torch.zeros_like(trans) if self.bound else None
            tabs = torch.zeros_like(trans) if self.bound else None
            for m, name in enumerate(['coord_mlp', 'cross_product_mlp'][:nm]):
                W1 = sd[f'{q}.{name}.0.weight']
                u, eu, d2 = self._first_layer(S, W1, None, P[:, m * H:(m + 1) * H],
                                              P[:, nm * H + m * H:nm * H + (m + 1) * H], r, c, x, d0[sl])
                mm_, em = self._mlp2(u, eu, sd[f'{q}.{name}.2.weight'], sd[f'{q}.{name}.2.bias'], self.ar_coord)
                phi = mm_ @ w3
                if m == 0:
                    diff = x[r] - x[c]
                    den = torch.sqrt(d2 + 1e-8) + nc
                    dvec = diff / den
                    edir = 16 * U * dvec.abs() if self.bound else None
                else:
                    av, bv = x[r] - cent[gid[r]], x[c] - cent[gid[c]]
                    cr = torch.cross(av, bv, dim=1)
                    cn = torch.linalg.norm(cr, dim=1, keepdim=True) + nc
                    dvec = cr / cn
                    if self.bound:
                        p1 = torch.stack([av[:, 1] * bv[:, 2], av[:, 2] * bv[:, 0], av[:, 0] * bv[:, 1]], 1).abs()
                        p2 = torch.stack([av[:, 2] * bv[:, 1], av[:, 0] * bv[:, 2], av[:, 1] * bv[:, 0]], 1).abs()
                        ecr = 5 * U * (p1 + p2)
                        ecn = ecr.sum(1, keepdim=True) + 6 * U * cn
                        edir = ecr / cn + cr.abs() * ecn / cn ** 2 + U * dvec.abs()
                f = torch.tanh(phi) * rng if cfg.tanh else phi
                if self.bound:
                    ephi = em @ w3.abs() + gam(H + 2) * (mm_.abs() @ w3.abs())
                    ef = (rng * (ephi + 2.0 ** -21) + 2 * U * f.abs()) if cfg.tanh else ephi
                    et = et + dvec.abs() * ef[:, None] + f.abs()[:, None] * edir + 2 * U * (dvec * f[:, None]).abs()
                    tabs = tabs + (dvec * f[:, None]).abs()
                trans = trans + dvec * f[:, None]
            xagg.index_add_(0, r, trans)
            if self.bound:
                ex.index_add_(0, r, et)
                sabs.index_add_(0, r, tabs)
        if self.bound:
            deg = torch.bincount(er, minlength=N).to(self.dtype)[:, None] * nm
            ex = ex + (deg + 2) * U / (1 - (deg + 2) * U) * sabs
        return {'xagg': (xagg[:self.n_coord_rows], ex[:self.n_coord_rows] if self.bound else None)}

    def _graph_rows(self, S):
        ma, mr = self.inp[3].to(self.device), self.inp[4].to(self.device)
        return torch.cat([ma, mr]).long()

    def _centroid(self, x, ex, gid):
        B = self.dm.B
        cnt = torch.bincount(gid, minlength=B).clamp(min=1).to(self.dtype)[:, None]
        c = torch.zeros((B, 3), dtype=self.dtype, device=self.device).index_add_(0, gid, x) / cnt
        if not self.bound:
            return c, None
        sa = torch.zeros_like(c).index_add_(0, gid, x.abs())
        es = torch.zeros_like(c).index_add_(0, gid, ex) if ex is not None else 0.0
        n = cnt
        return c, (es + (n + 8) * U / (1 - (n + 8) * U) * sa) / cnt + U * c.abs()

    def centroid(self, S, x_old):
        gid = self._graph_rows(S)
        c, e = self._centroid(self.t(S[x_old][:, :3]), None, gid)
        return {'cent': (c, e)}

    def finish(self, S, l, x_old, x_new):
        cfg = self.cfg
        x = self.t(S[x_old][:, :3])
        xa = self.t(S['xagg'][:, :3])
        n = self.n_coord_rows
        if cfg.aggregation_method == 'mean':
            div = self.t(S['deg'][:n]).clamp(min=1)[:, None]
        else:
            div = cfg.normalization_factor
        upd = xa[:n] / div
        xn = x.clone()
        xn[:n] = x[:n] + upd
        exn = None
        if self.bound:
            exn = torch.zeros_like(xn)
            exn[:n] = U * upd.abs() + U * xn[:n].abs()
        gid = self._graph_rows(S)
        c, ec = self._centroid(xn, exn, gid)
        return {x_new: (xn, exn), 'cent': (c, ec), 'xagg': (torch.zeros_like(xa), None)}

    def post(self, S, x_old):
        """Outputs of the forward: velocity (joint: per-graph mean removed) | decoders(embedding_out(h)), folded pairs."""
        cfg, sd, dm = self.cfg, self.sd, self.dm
        J = cfg.joint_nf
        h = self.t(S['h'])
        xf, xi = self.t(S[x_old][:, :3]), self.t(S['x_in'][:, :3])
        vel = xf - xi
        ev = U * vel.abs() if self.bound else None
        if cfg.update_pocket_coords:
            gid = self._graph_rows(S)
            vm, evm = self._centroid(vel, ev, gid)
            vel = vel - vm[gid]
            if self.bound:
                ev = ev + evm[gid] + U * vel.abs()
        outs = []
        for lo, hi, dec in ((0, dm.NL, 'atom_decoder'), (dm.NL, dm.N, 'residue_decoder')):
            Wd = sd[dec + '.0.weight'] @ sd['egnn.embedding_out.weight'][:J]
            bd = sd[dec + '.0.bias'] + sd[dec + '.0.weight'] @ sd['egnn.embedding_out.bias'][:J]
            z, ez = linear_b(h[lo:hi], self._e(h[lo:hi]), Wd, bd, self.ar_ffma)
            if self.bound:
                ez = ez + U * (h[lo:hi].abs() @ Wd.abs().T + bd.abs())
                hid, eh = silu_b(z, ez)
            else:
                hid, eh = F.silu(z), None
            o, eo = linear_b(hid, eh, sd[dec + '.2.weight'], sd[dec + '.2.bias'], self.ar_ffma)
            val = torch.cat([vel[lo:hi], o], 1)
            err = torch.cat([ev[lo:hi], eo], 1) if self.bound else None
            outs.append((val, err))
        return {'out_atoms': outs[0], 'out_residues': outs[1]}

    def run(self, op: Op, S):
        k = op.kind
        if k == 'prep':
            return self.prep(S)
        if k in ('g1', 'g2', 'g3'):
            return getattr(self, k)(S, op.layer, op.sub)
        if k == 'gcl':
            return self.gcl(S, op.layer, op.sub, op.x_old)
        if k == 'g4':
            return self.g4(S, op.layer)
        if k == 'coord':
            return self.coord(S, op.layer, op.x_old)
        if k == 'finish':
            return self.finish(S, op.layer, op.x_old, op.x_new)
        if k == 'centroid':
            return self.centroid(S, op.x_old)
        if k in ('velmean', 'post'):
            return self.post(S, op.x_old)
        raise KeyError(k)


def output_view(S, name, entry):
    """The part of state S a restatement output refers to (P: its column block)."""
    if name == 'P':
        return S['P'][:, entry[2]]
    if name in ('x_in', 'x_ping', 'x_pong', 'xagg', 'cent'):
        n = entry[0].shape[0]
        return S[name][:n, :3]
    return S[name]


def dead_p_mask(cfg, dm: Dims, mode, n_cols):
    """Conditional mode: elements of the merged first-layer GEMM's output that the kernel skips (tiles of pocket rows x
    receiver-side coordinate columns): 128 x H tiles on wgmma, 128 x 128 tiles in the fp32 kernel."""
    mask = torch.zeros((dm.N, n_cols), dtype=torch.bool)
    if cfg.update_pocket_coords:
        return mask
    nrecv = nm_of(cfg) * cfg.hidden_nf
    tn = cfg.hidden_nf if (effective_mode(cfg, mode) & 1) else 128
    r0 = -(-dm.NL // 128) * 128
    c1 = (nrecv // tn) * tn
    mask[r0:, :c1] = True
    return mask


# ---- CPU emulation: the restatements chained into a whole forward (fp32 or fp64) -------------------------------------
def initial_state(cfg, inputs, dtype=torch.float32):
    """The state the first checked launch needs, built like plan / edges do (oracle edge list, CSR order)."""
    from oracle import egnn_oracle
    xa, xr, t, ma, mr = inputs
    N, H = len(ma) + len(mr), cfg.hidden_nf
    edges = egnn_oracle.build_edges(cfg, ma, mr, xa[:, :3], xr[:, :3])
    er, ec = edges[0], edges[1]
    x = torch.cat([xa[:, :3], xr[:, :3]], 0).to(torch.float32)
    x4 = torch.cat([x, torch.zeros(N, 1)], 1)
    diff = x.to(dtype)[er] - x.to(dtype)[ec]
    deg = torch.bincount(er, minlength=N)
    ldp = (2 * nm_of(cfg) + 2) * H
    S = {'x_in': x4.clone(), 'x_ping': torch.zeros(N, 4), 'x_pong': torch.zeros(N, 4), 'xagg': torch.zeros(N, 4),
         'h': torch.zeros(N, H), 'hT': torch.zeros(N, H), 'agg': torch.zeros(N, H), 'P': torch.zeros(N, ldp),
         'cent': torch.zeros(max(int(torch.cat([ma, mr]).max()) + 1, t.numel() if cfg.condition_time else 0), 4),
         'deg': deg.to(torch.int32), 'row_ptr': torch.cat([torch.zeros(1, dtype=torch.int64), deg.cumsum(0)]).to(torch.int32),
         'gid': torch.cat([ma, mr]).to(torch.int32), 'erow': er.to(torch.int32), 'ecol': ec.to(torch.int32),
         'ed0': (diff * diff).sum(1)}
    S['velmean'] = torch.zeros_like(S['cent'])
    return {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in S.items()}


def apply(S, outs):
    for name, entry in outs.items():
        val = entry[0]
        if name in ('out_atoms', 'out_residues'):
            S[name] = val
            continue
        dst = output_view(S, name, entry)
        dst.copy_(val.to(dst.dtype))


def emulate(cfg, sd, inputs, mode=0, dtype=torch.float32):
    """The whole forward from the restatements alone (what the kernels compute, launch by launch)."""
    S = initial_state(cfg, inputs, dtype)
    R = Restater(cfg, sd, inputs, mode, dtype)
    for _, _, op in launch_units(cfg, False):
        apply(S, R.run(op, S))
    return S['out_atoms'], S['out_residues']


# ---- the binade-sweep case ---------------------------------------------------------------------------------------
SWEEP_CFG = DynamicsConfig(hidden_nf=128, joint_nf=32, n_layers=2, inv_sublayers=1)
SWEEP_GRAPHS = ([12, 20, 7], [60, 90, 40])
SWEEP_H_EXP = (-20, 15)          # embedding output channel c is scaled by 2^e_c, e_c spread evenly over this range
SWEEP_U_EXP = (-26, 3)           # first-layer output unit j of every edge / coordinate MLP is scaled by 2^f_j


def binade_sweep_case(seed=7):
    """(cfg, state_dict, inputs): a seeded state dict whose embedding rows and first-layer rows are scaled by powers of
    two, column by column of their outputs, so that the A operands of the first-layer GEMMs (h), of the node MLP
    ([h | agg / 100]) and of the edge kernels (SiLU of the first layer) spread from about 2^-20 to 2^14: through the fp16
    subnormal range (< 2^-14), below the fp16 limit."""
    cfg = SWEEP_CFG
    sd = syn.synthetic_state_dict(cfg, seed)
    H = cfg.hidden_nf
    e = torch.round(torch.linspace(*SWEEP_H_EXP, H)).to(torch.float64)
    sh = torch.pow(2.0, e[torch.randperm(H, generator=torch.Generator().manual_seed(seed))]).to(torch.float32)
    sd['egnn.embedding.weight'] = sd['egnn.embedding.weight'] * sh[:, None]
    sd['egnn.embedding.bias'] = sd['egnn.embedding.bias'] * sh
    f = torch.pow(2.0, torch.round(torch.linspace(*SWEEP_U_EXP, H)).to(torch.float64)).to(torch.float32)
    for k in list(sd):
        if k.endswith(('edge_mlp.0.weight', 'coord_mlp.0.weight', 'cross_product_mlp.0.weight')):
            sd[k] = sd[k] * f[:, None]
            sd[k[:-len('weight')] + 'bias'] = sd[k[:-len('weight')] + 'bias'] * f
    inputs = syn.synthetic_denoiser_inputs(cfg, *SWEEP_GRAPHS, seed=seed)
    return cfg, sd, inputs


def sweep_operand_ranges(cfg, sd, inputs):
    """min / max |A| over the nonzero A operands of the first g1, g2 and GCL edge kernel of the sweep case (float64)."""
    S = initial_state(cfg, inputs, torch.float64)
    R = Restater(cfg, sd, inputs, 0, torch.float64)
    R.bound = False
    apply(S, R.prep(S))
    apply(S, R.g1(S, 0, 0))
    er, ec = S['erow'].long(), S['ecol'].long()
    H, nq = cfg.hidden_nf, R.nq
    u, _, _ = R._first_layer(S, sd['egnn.e_block_0.gcl_0.edge_mlp.0.weight'].double(), None, S['P'][:, nq:nq + H],
                             S['P'][:, nq + H:nq + 2 * H], er, ec, S['x_in'][:, :3], S['ed0'])
    apply(S, R.gcl(S, 0, 0, 'x_in'))

    def rng(a):
        a = a.abs()
        a = a[a > 0]
        return float(a.min()), float(a.max())
    return {'g1': rng(S['h']), 'g2': rng(torch.cat([S['h'], S['agg'] / cfg.normalization_factor], 1)),
            'gcl': rng(F.silu(u))}


# ---- cases ------------------------------------------------------------------------------------------------------
def configs2_case():
    cfg = FULLATOM_COND
    return cfg, syn.synthetic_state_dict(cfg, 0), syn.synthetic_denoiser_inputs(cfg, [25] * 64, [175] * 64, seed=3)


# bench.py's 'moad' workload (configs/moad_fullatom_cond.yml): hidden_nf 192 with the edge-type table
MOAD_COND = FULLATOM_COND.with_(hidden_nf=192, edge_embedding_dim=8, edge_cutoff_pocket=4.0, edge_cutoff_interaction=7.0)


def moad_case():
    cfg = MOAD_COND
    return cfg, syn.synthetic_state_dict(cfg, 0), syn.synthetic_denoiser_inputs(cfg, [25] * 64, [175] * 64, seed=3)


# ---- the tensor-core kernel instances a forward launches ------------------------------------------------------------
TC_FORMATS = ('TF32x3', 'F16x3', 'F16x1')          # TcFormat enumerators, in order (dsb_internal.cuh)


def tc_instances(cfg, mode, det):
    """{(kernel, COORD, FMT, H, TB, DET)} of the tensor-core kernels one forward launches, following dsb_dynamics_forward
    and launch_tc_node_gemm / launch_tc_edge_gcl / launch_tc_edge_coord: mode bits 1 / 2 / 4 put the node GEMMs / GCL edge
    kernel / coordinate edge kernel on wgmma, bits 8 / 16 pick the format, an edge-type table (edge_embedding_dim > 0)
    selects TB.  The node GEMM is templated on FMT and H only: its COORD, TB and DET are None."""
    mm = effective_mode(cfg, mode)
    fmt = TC_FORMATS[0] if not mm & 8 else TC_FORMATS[2] if mm & 16 else TC_FORMATS[1]
    H, tb, det = cfg.hidden_nf, bool(cfg.edge_embedding_dim), bool(det)
    out = set()
    if mm & 1:
        out.add(('tc_node_gemm_kernel', None, fmt, H, None, None))
    for bit, coord in ((2, False), (4, True)):
        if mm & bit:
            out.add(('tc_edge_kernel', coord, fmt, H, tb, det))
    return out


def _template_arg(s):
    """One demangled template argument: '(bool)1' / 'true', '(int)192' / '192', '(dsb::TcFormat)1' / 'dsb::TcFormat::F16x3'."""
    s = s.strip()
    if s.startswith('('):
        typ, val = s[1:].split(')', 1)
        if typ == 'bool':
            return bool(int(val))
        if typ.endswith('TcFormat'):
            return TC_FORMATS[int(val)]
        return int(val)
    if s in ('true', 'false'):
        return s == 'true'
    if 'TcFormat::' in s:
        name = s.rsplit('::', 1)[1]
        assert name in TC_FORMATS, s
        return name
    return int(s)


def demangle(names):
    """Demangled forms of kernel names (cu++filt from the CUDA toolkit; names that are not mangled pass unchanged)."""
    names = list(names)
    mangled = [n for n in names if n.startswith('_Z')]
    if not mangled:
        return names
    import shutil
    import subprocess
    filt = shutil.which('cu++filt') or '/usr/local/cuda/bin/cu++filt'
    out = subprocess.run([filt], input='\n'.join(mangled) + '\n', capture_output=True, text=True, check=True).stdout
    table = dict(zip(mangled, out.splitlines()))
    return [table.get(n, n) for n in names]


def parse_tc_instance(name):
    """(kernel, COORD, FMT, H, TB, DET) of a demangled tensor-core kernel name, None for any other kernel."""
    for kernel in ('tc_node_gemm_kernel', 'tc_edge_kernel'):
        i = name.find(kernel + '<')
        if i < 0:
            continue
        args = [_template_arg(a) for a in name[i + len(kernel) + 1:name.index('>', i)].split(',')]
        if kernel == 'tc_node_gemm_kernel':
            fmt, H = args
            return kernel, None, fmt, H, None, None
        coord, fmt, H, tb = args[:4]
        det = args[4] if len(args) > 4 else False        # DET = false is a default argument: it may be left out
        return kernel, coord, fmt, H, tb, det
    return None
