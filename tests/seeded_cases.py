"""numpy restatement of the seeded generator dsb_seeded_normal (include/diffsbdd_b200.h): Philox4x32-10, the counter
layout (column group, row within the graph, role | draw_hi << 4, draw_lo) and the Box-Muller / uniform mappings."""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
ROLE_LIGAND, ROLE_POCKET, ROLE_JOINT_X, ROLE_GRAPH = 0, 1, 2, 3


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Vectorised over equal-shape uint32 arrays; returns the four output words as uint64 arrays holding uint32 values."""
    c = [np.asarray(v, dtype=np.uint64) & 0xFFFFFFFF for v in (c0, c1, c2, c3)]
    k0 = np.asarray(k0, dtype=np.uint64) & 0xFFFFFFFF
    k1 = np.asarray(k1, dtype=np.uint64) & 0xFFFFFFFF
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = c[0] * np.uint64(M0)
        p1 = c[2] * np.uint64(M1)
        hi0, lo0 = p0 >> np.uint64(32), p0 & mask
        hi1, lo1 = p1 >> np.uint64(32), p1 & mask
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(W0)) & mask
        k1 = (k1 + np.uint64(W1)) & mask
    return c


def local_rows(role, lig_mask, pocket_mask, n_graphs):
    """(graph, index within the graph) of every output row of ``role``."""
    lig_mask, pocket_mask = np.asarray(lig_mask), np.asarray(pocket_mask)

    def within(mask):
        starts = np.searchsorted(mask, np.arange(n_graphs))
        return mask, np.arange(len(mask)) - starts[mask]
    if role == ROLE_LIGAND:
        return within(lig_mask)
    if role == ROLE_POCKET:
        return within(pocket_mask)
    if role == ROLE_GRAPH:
        return np.arange(n_graphs), np.zeros(n_graphs, dtype=np.int64)
    gl, il = within(lig_mask)
    gp, ip = within(pocket_mask)
    n_lig = np.bincount(lig_mask, minlength=n_graphs)
    return np.concatenate([gl, gp]), np.concatenate([il, ip + n_lig[gp]])


def words(role, cols, seeds, draw, lig_mask, pocket_mask):
    """Raw words [rows, 4 * ceil(cols / 4)] (uint32) as the kernel's DSB_RNG_BITS output before the column cut."""
    seeds = np.asarray(seeds, dtype=np.uint64)
    g, i = local_rows(role, lig_mask, pocket_mask, len(seeds))
    groups = (cols + 3) // 4
    gg = np.repeat(g, groups)
    ii = np.repeat(i, groups).astype(np.uint64)
    jj = np.tile(np.arange(groups, dtype=np.uint64), len(g))
    draw = int(draw)
    c2 = np.full_like(jj, role | ((draw >> 32) << 4))
    c3 = np.full_like(jj, draw & 0xFFFFFFFF)
    w = philox4x32_10(jj, ii, c2, c3, seeds[gg], seeds[gg] >> np.uint64(32))
    return np.stack(w, axis=1).reshape(len(g), 4 * groups).astype(np.uint32)


def uniform(w):
    """U(w) = fmaf((float)w, 2^-32, 2^-33): exact fp32 restatement ((float)w * 2^-32 is exact, one rounding of the add)."""
    return np.float32(w.astype(np.float32) * np.float32(2.0 ** -32)) + np.float32(2.0 ** -33)


def normals(w):
    """Box-Muller in float64 on the fp32 inputs the kernel uses; the kernel's fp32 logf / sqrtf / sincospif stay within a
    few ulp of this."""
    u = uniform(w[:, 0::2]).astype(np.float64)
    v = (w[:, 1::2].astype(np.float32) * np.float32(2.0 ** -32)).astype(np.float64)
    r = np.sqrt(-2.0 * np.log(u))
    out = np.empty(w.shape, dtype=np.float64)
    out[:, 0::2] = r * np.cos(2 * np.pi * v)
    out[:, 1::2] = r * np.sin(2 * np.pi * v)
    return out


def expected_sizes(prob, n_pocket, u):
    """Inverse CDF of p(n_lig | n_pocket): the smallest i with u <= cdf[i] (cdf normalised to end at 1)."""
    prob = np.asarray(prob, dtype=np.float64)
    out = []
    for j, uu in zip(np.asarray(n_pocket), np.asarray(u, dtype=np.float64)):
        cdf = np.cumsum(prob[:, j])
        cdf = cdf / cdf[-1]
        out.append(min(int(np.searchsorted(cdf, uu, side='left')), prob.shape[0] - 1))
    return np.array(out)
