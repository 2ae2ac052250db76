// Node-level kernels of the denoiser: graph plan, encoders+embedding, cut-off edge list (CSR), the
// node GEMM (factorised first layers / node MLP), coordinate finish + centroid, decoders.
// Reference semantics: equivariant_diffusion/dynamics.py:87-187, egnn_new.py:48-58, :225-244, :305-316.
#include "dsb_internal.cuh"

namespace dsb {

// =====================================================================================================
// plan: per-graph node ranges from the sorted int64 masks (utils.py:146-154 builds them with
// repeat_interleave, so they are non-decreasing).
// =====================================================================================================
// One pass over both masks: element i starts graphs (mask[i-1], mask[i]] (several when graphs in between are empty); the
// ends are written by the threads next to them.  (A binary search per graph is 14 dependent global loads: 13.6 us for 65
// threads; this is one coalesced load per element.)
__device__ __forceinline__ void plan_one(const int64_t* __restrict__ mask, int n, int B, int32_t* __restrict__ off, int i) {
  if (n == 0) { if (i <= B) off[i] = 0; return; }
  if (i >= n) return;
  const int64_t cur = mask[i];
  const int64_t prev = i > 0 ? mask[i - 1] : -1;
  for (int64_t g = prev + 1; g <= cur; ++g) off[g] = i;          // graphs prev+1 .. cur start here
  if (i == n - 1) for (int64_t g = cur + 1; g <= B; ++g) off[g] = n;     // trailing empty graphs and the end marker
}

__global__ void plan_kernel(const int64_t* __restrict__ mask_atoms, const int64_t* __restrict__ mask_res,
                            int NL, int NP, int B, int32_t* __restrict__ lig_off,
                            int32_t* __restrict__ poc_off) {
  pdl_trigger();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  plan_one(mask_atoms, NL, B, lig_off, i);
  plan_one(mask_res, NP, B, poc_off, i);
}

int launch_plan(const dsb_dynamics* d, const Dims& dm, const Workspace& ws, const int64_t* mask_atoms,
                const int64_t* mask_residues, cudaStream_t s) {
  const int n = max(max(dm.NL, dm.NP), dm.B + 1);
  int threads = 256, blocks = (n + threads - 1) / threads;
  DSB_CUDA_OK(launch_k(plan_kernel, blocks, threads, 0, s, mask_atoms, mask_residues, dm.NL, dm.NP, dm.B, ws.lig_off, ws.poc_off));
  return 0;
}

// =====================================================================================================
// prep: x/h split, atom/residue encoder (Linear-SiLU-Linear), time channel, embedding Linear(J+1 -> H)
// (dynamics.py:89-111, egnn_new.py:233).  The encoder's second Linear and the embedding are both affine
// with nothing in between, so they are folded at pack time into one [2F+1][H] matrix per node type
// (rows: encoder hidden units, last row: the time column of the embedding) -- 2F+1 MACs per output instead
// of 2F*J + (J+1).  One CTA = 32 nodes of one type; thread = output column.
// =====================================================================================================
constexpr int PREP_NODES = 32;
constexpr int PREP_THREADS = 256;

struct PrepArgs {
  const float* xh_atoms; const float* xh_res; const float* t; int t_numel;
  const int64_t* mask_atoms; const int64_t* mask_res;
  int NL, NP, A, R, H; int cond_time; int coords_only;
  const float *aenc0_w, *aenc0_b, *renc0_w, *renc0_b;
  const float *pre_wT[2], *pre_b[2];
  int32_t* gid; float4* x0; float* h;
};

__global__ void __launch_bounds__(PREP_THREADS) prep_kernel(PrepArgs p) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ __align__(16) float sm[];
  const int lig_blocks = (p.NL + PREP_NODES - 1) / PREP_NODES;
  const bool is_lig = blockIdx.x < lig_blocks;
  const int F = is_lig ? p.A : p.R;
  const int F2 = 2 * F;
  const int base = is_lig ? blockIdx.x * PREP_NODES : (blockIdx.x - lig_blocks) * PREP_NODES;
  const int count = is_lig ? p.NL : p.NP;
  const int nn = min(PREP_NODES, count - base);
  const float* xh = is_lig ? p.xh_atoms : p.xh_res;
  const int64_t* mask = is_lig ? p.mask_atoms : p.mask_res;
  const int ld = 3 + F;
  const int node0 = is_lig ? base : p.NL + base;
  const float *w0 = is_lig ? p.aenc0_w : p.renc0_w, *b0 = is_lig ? p.aenc0_b : p.renc0_b;
  const float* wT = p.pre_wT[is_lig ? 0 : 1];
  const float* bf = p.pre_b[is_lig ? 0 : 1];

  float* s_f = sm;                                 // [32][F]
  float* s_hid = s_f + PREP_NODES * F;             // [2F + 1][32]  k-major; last row = t of the node's graph
  const int tid = threadIdx.x;

  for (int i = tid; i < nn; i += PREP_THREADS) {
    const float* row = xh + (size_t)(base + i) * ld;
    p.x0[node0 + i] = make_float4(row[0], row[1], row[2], 0.f);
    p.gid[node0 + i] = (int)mask[base + i];
  }
  if (p.coords_only) return;
  for (int i = tid; i < PREP_NODES * F; i += PREP_THREADS) {
    const int n = i / F, k = i - n * F;
    s_f[i] = n < nn ? xh[(size_t)(base + n) * ld + 3 + k] : 0.f;
  }
  __syncthreads();
  for (int i = tid; i < PREP_NODES * F2; i += PREP_THREADS) {
    const int n = i & (PREP_NODES - 1), o = i >> 5;
    float acc = b0[o];
    for (int k = 0; k < F; ++k) acc = fmaf(s_f[n * F + k], w0[o * F + k], acc);
    s_hid[i] = silu_f(acc);
  }
  if (p.cond_time && tid < PREP_NODES)              // time channel (dynamics.py:104-111)
    s_hid[F2 * PREP_NODES + tid] = tid < nn ? ((p.t_numel == 1) ? p.t[0] : p.t[(int)mask[base + tid]]) : 0.f;
  __syncthreads();
  const int K = F2 + (p.cond_time ? 1 : 0);
  for (int c = tid; c < p.H; c += PREP_THREADS) {
    const float bias = bf[c];
#pragma unroll 1
    for (int n0 = 0; n0 < nn; n0 += 8) {
      float acc[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = bias;
      for (int k = 0; k < K; ++k) {
        const float w = __ldg(wT + (size_t)k * p.H + c);
        const float4 ha = *reinterpret_cast<const float4*>(s_hid + k * PREP_NODES + n0);
        const float4 hb = *reinterpret_cast<const float4*>(s_hid + k * PREP_NODES + n0 + 4);
        acc[0] = fmaf(ha.x, w, acc[0]); acc[1] = fmaf(ha.y, w, acc[1]); acc[2] = fmaf(ha.z, w, acc[2]); acc[3] = fmaf(ha.w, w, acc[3]);
        acc[4] = fmaf(hb.x, w, acc[4]); acc[5] = fmaf(hb.y, w, acc[5]); acc[6] = fmaf(hb.z, w, acc[6]); acc[7] = fmaf(hb.w, w, acc[7]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (n0 + j < nn) p.h[(size_t)(node0 + n0 + j) * p.H + c] = acc[j];
    }
  }
}

int launch_prep(const dsb_dynamics* d, const Dims& dm, const Workspace& ws, const float* xh_atoms,
                const float* xh_residues, const float* t, int64_t t_numel, const int64_t* mask_atoms,
                const int64_t* mask_residues, bool coords_only, cudaStream_t s) {
  const dsb_config& c = d->cfg;
  PrepArgs p;
  p.xh_atoms = xh_atoms; p.xh_res = xh_residues; p.t = t; p.t_numel = (int)t_numel;
  p.mask_atoms = mask_atoms; p.mask_res = mask_residues;
  p.NL = dm.NL; p.NP = dm.NP; p.A = c.atom_nf; p.R = c.residue_nf;
  p.H = c.hidden_nf; p.cond_time = c.condition_time;
  p.coords_only = coords_only ? 1 : 0;
  const PackedWeights& w = d->w;
  p.aenc0_w = w.aenc0_w; p.aenc0_b = w.aenc0_b; p.renc0_w = w.renc0_w; p.renc0_b = w.renc0_b;
  p.pre_wT[0] = w.pre_wT[0]; p.pre_wT[1] = w.pre_wT[1]; p.pre_b[0] = w.pre_b[0]; p.pre_b[1] = w.pre_b[1];
  p.gid = ws.gid; p.x0 = ws.xbuf[0]; p.h = ws.h;
  int Fm = c.atom_nf > c.residue_nf ? c.atom_nf : c.residue_nf;
  size_t smem = sizeof(float) * PREP_NODES * (size_t)(3 * Fm + 1);
  int blocks = (dm.NL + PREP_NODES - 1) / PREP_NODES + (dm.NP + PREP_NODES - 1) / PREP_NODES;
  if (blocks == 0) return 0;
  DSB_CUDA_OK(launch_k(prep_kernel, blocks, PREP_THREADS, smem, s, p));
  return 0;
}

// =====================================================================================================
// edges: dynamics.py:169-187.  Row i's neighbours = ligand nodes of its graph, then pocket nodes of its
// graph (ascending global index == the reference's torch.where row-major order), each filtered by the
// cut-off of the (row type, col type) block.  One warp per row; count -> scan -> fill.
// =====================================================================================================
struct EdgeBuildArgs {
  const float4* x; const int32_t* gid; const int32_t* lig_off; const int32_t* poc_off;
  int NL, N; float cut_l, cut_p, cut_i;
  int32_t* deg; const int32_t* row_ptr; int32_t* erow; int32_t* ecol; float* ed0; int64_t Ecap;
  const int32_t* vrow_ptr; int32_t* vmap;
};

template <bool FILL>
__global__ void __launch_bounds__(256) edge_rows_kernel(EdgeBuildArgs a) {
  pdl_trigger();
  pdl_wait();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= a.N) return;
  const int i = warp;
  const int g = a.gid[i];
  const bool lig_i = i < a.NL;
  const float4 xi = a.x[i];
  int count = 0;
  const int base = FILL ? a.row_ptr[i] : 0;
  const int vbase = FILL ? a.vrow_ptr[i] : 0;
#pragma unroll 1
  for (int part = 0; part < 2; ++part) {
    const int lo = part == 0 ? a.lig_off[g] : a.NL + a.poc_off[g];
    const int hi = part == 0 ? a.lig_off[g + 1] : a.NL + a.poc_off[g + 1];
    const float cut = part == 0 ? (lig_i ? a.cut_l : a.cut_i) : (lig_i ? a.cut_i : a.cut_p);
    for (int j0 = lo; j0 < hi; j0 += 32) {
      const int j = j0 + lane;
      bool keep = false;
      float d2 = 0.f;
      if (j < hi) {
        const float4 xj = a.x[j];
        const float dx = xi.x - xj.x, dy = xi.y - xj.y, dz = xi.z - xj.z;
        d2 = dx * dx + dy * dy + dz * dz;
        keep = (cut < 0.f) || (sqrtf(d2) <= cut);
      }
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (FILL && keep) {
        const int k = count + __popc(m & ((1u << lane) - 1u));
        const int64_t e = (int64_t)base + k;
        if (e < a.Ecap) { a.erow[e] = i; a.ecol[e] = j; a.ed0[e] = d2; a.vmap[vbase + k] = (int32_t)e; }
      }
      count += __popc(m);
    }
  }
  if (!FILL && lane == 0) a.deg[i] = count;
  if (FILL) {       // pad rows of this receiver's segment in the virtual order
    const int padded = (count + kRowChunk - 1) / kRowChunk * kRowChunk;
    if (count + lane < padded && (int64_t)base + count <= a.Ecap) a.vmap[vbase + count + lane] = -1;
  }
}

// exclusive scans of deg[0..N) -> row_ptr[0..N] and of the chunk-padded degrees -> vrow_ptr[0..N]; single CTA (N is ~1e4).
// Every thread owns SCAN_PER consecutive elements (all loads of a pass in flight together, a serial scan in registers), one
// warp-shuffle scan of the thread sums and one of the warp sums per pass: N = 12 800 is one pass instead of 13 block scans.
constexpr int SCAN_PER = 16;
__global__ void __launch_bounds__(1024) scan_kernel(const int32_t* __restrict__ deg, int32_t* __restrict__ row_ptr,
                                                     int32_t* __restrict__ vrow_ptr, int N, int64_t Ecap,
                                                     int32_t* __restrict__ status) {
  pdl_trigger();
  pdl_wait();
  __shared__ int s_warp[2][32];
  __shared__ int s_carry[2];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid < 2) s_carry[tid] = 0;
  __syncthreads();
  for (int base = 0; base < N; base += 1024 * SCAN_PER) {
    const int i0 = base + tid * SCAN_PER;
    int v[SCAN_PER];
#pragma unroll
    for (int k = 0; k < SCAN_PER; ++k) v[k] = i0 + k < N ? deg[i0 + k] : 0;
    int x = 0, y = 0;
#pragma unroll
    for (int k = 0; k < SCAN_PER; ++k) { x += v[k]; y += (v[k] + kRowChunk - 1) / kRowChunk * kRowChunk; }
    const int tx = x, ty = y;                    // this thread's totals
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int a = __shfl_up_sync(0xffffffffu, x, o), b = __shfl_up_sync(0xffffffffu, y, o);
      if (lane >= o) { x += a; y += b; }
    }
    if (lane == 31) { s_warp[0][wid] = x; s_warp[1][wid] = y; }
    __syncthreads();
    if (wid < 2) {
      int w = s_warp[wid][lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int a = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += a; }
      s_warp[wid][lane] = w;
    }
    __syncthreads();
    int ex = x - tx + (wid > 0 ? s_warp[0][wid - 1] : 0) + s_carry[0];        // exclusive prefix of this thread's first element
    int vex = y - ty + (wid > 0 ? s_warp[1][wid - 1] : 0) + s_carry[1];
#pragma unroll
    for (int k = 0; k < SCAN_PER; ++k) {
      if (i0 + k < N) { row_ptr[i0 + k] = ex; vrow_ptr[i0 + k] = vex; }
      ex += v[k]; vex += (v[k] + kRowChunk - 1) / kRowChunk * kRowChunk;
    }
    __syncthreads();
    if (tid == 1023) { s_carry[0] = ex; s_carry[1] = vex; }
    __syncthreads();
  }
  if (tid == 0) {
    const int E = s_carry[0];
    row_ptr[N] = E;
    vrow_ptr[N] = s_carry[1];
    if (status) {
      status[1] = E;
      if ((int64_t)E > Ecap) atomicOr(&status[2], 1);
    }
  }
}

int launch_edges(const dsb_dynamics* d, const Dims& dm, const Workspace& ws, int32_t* status, cudaStream_t s,
                 int max_launches) {
  const dsb_config& c = d->cfg;
  EdgeBuildArgs a;
  a.x = ws.xbuf[0]; a.gid = ws.gid; a.lig_off = ws.lig_off; a.poc_off = ws.poc_off;
  a.NL = dm.NL; a.N = dm.N; a.cut_l = c.edge_cutoff_ligand; a.cut_p = c.edge_cutoff_pocket;
  a.cut_i = c.edge_cutoff_interaction;
  a.deg = ws.deg; a.row_ptr = ws.row_ptr; a.erow = ws.erow; a.ecol = ws.ecol; a.ed0 = ws.ed0; a.Ecap = dm.Ecap;
  a.vrow_ptr = ws.vrow_ptr; a.vmap = ws.vmap;
  const int blocks = (dm.N * 32 + 255) / 256;
  if (dm.N == 0) return 0;
  if (max_launches > 0) DSB_CUDA_OK(launch_k(edge_rows_kernel<false>, blocks, 256, 0, s, a));
  if (max_launches > 1) DSB_CUDA_OK(launch_k(scan_kernel, 1, 1024, 0, s, ws.deg, ws.row_ptr, ws.vrow_ptr, dm.N, dm.Ecap, status));
  if (max_launches > 2) DSB_CUDA_OK(launch_k(edge_rows_kernel<true>, blocks, 256, 0, s, a));
  DSB_CUDA_OK(cudaGetLastError());
  return 0;
}

// =====================================================================================================
// coordinate finish + per-graph centroid.  x_new = x_old + mask * (sum_j trans_ij) / normalization_factor
// (egnn_new.py:114-121) and the centroid over ALL nodes of the graph used by coord2cross
// (egnn_new.py:307-310).  One CTA per graph.
// =====================================================================================================
__global__ void __launch_bounds__(128) coord_finish_kernel(const float4* __restrict__ x_old, float4* __restrict__ x_new,
                                                            float4* __restrict__ xagg, const int32_t* __restrict__ lig_off,
                                                            const int32_t* __restrict__ poc_off, int NL, int n_coord_rows,
                                                            float norm, int apply_update, float4* __restrict__ cent,
                                                            const int32_t* __restrict__ deg) {
  pdl_trigger();
  pdl_wait();
  const int g = blockIdx.x;
  const int l0 = lig_off[g], l1 = lig_off[g + 1], p0 = NL + poc_off[g], p1 = NL + poc_off[g + 1];
  const int nl = l1 - l0, n = nl + (p1 - p0);
  float sx = 0.f, sy = 0.f, sz = 0.f;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const int i = k < nl ? l0 + k : p0 + (k - nl);
    float4 v = x_old[i];
    if (apply_update) {
      if (i < n_coord_rows) {
        const float4 a = xagg[i];
        xagg[i] = make_float4(0.f, 0.f, 0.f, 0.f);      // re-arm the accumulator for the next block
        const float dv = deg ? (float)max(deg[i], 1) : norm;          // 'mean' aggregation: the receiver's edge count
        v.x = v.x + __fdiv_rn(a.x, dv);
        v.y = v.y + __fdiv_rn(a.y, dv);
        v.z = v.z + __fdiv_rn(a.z, dv);
      }
      x_new[i] = v;
    }
    sx += v.x; sy += v.y; sz += v.z;
  }
  __shared__ float red[3][4];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sx += __shfl_xor_sync(0xffffffffu, sx, o);
    sy += __shfl_xor_sync(0xffffffffu, sy, o);
    sz += __shfl_xor_sync(0xffffffffu, sz, o);
  }
  const int wid = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[0][wid] = sx; red[1][wid] = sy; red[2][wid] = sz; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const float cnt = n > 0 ? (float)n : 1.f;
    float tx = red[0][0] + red[0][1] + red[0][2] + red[0][3];
    float ty = red[1][0] + red[1][1] + red[1][2] + red[1][3];
    float tz = red[2][0] + red[2][1] + red[2][2] + red[2][3];
    cent[g] = make_float4(tx / cnt, ty / cnt, tz / cnt, 0.f);
  }
}

int launch_coord_finish(const dsb_dynamics* d, const Dims& dm, const Workspace& ws, const float4* x_old,
                        float4* x_new, bool apply_update, cudaStream_t s) {
  if (dm.B == 0) return 0;
  DSB_CUDA_OK(launch_k(coord_finish_kernel, dm.B, 128, 0, s, x_old, x_new, ws.xagg, ws.lig_off, ws.poc_off, dm.NL,
                       dm.n_coord_rows, d->cfg.normalization_factor, apply_update ? 1 : 0, ws.cent,
                       d->cfg.aggregation_mean ? (const int32_t*)ws.deg : (const int32_t*)nullptr));
  return 0;
}

// =====================================================================================================
// post: embedding_out (H -> J+1, time channel dropped), atom/residue decoder, vel = x_final - x_in,
// NaN flag, joint-mode velocity mean removal (egnn_new.py:241; dynamics.py:136-167).
// =====================================================================================================
__global__ void __launch_bounds__(128) velmean_kernel(const float4* __restrict__ x_fin, const float4* __restrict__ x_in,
                                                       const int32_t* __restrict__ lig_off, const int32_t* __restrict__ poc_off,
                                                       int NL, float4* __restrict__ velmean) {
  pdl_trigger();
  pdl_wait();
  const int g = blockIdx.x;
  const int l0 = lig_off[g], l1 = lig_off[g + 1], p0 = NL + poc_off[g], p1 = NL + poc_off[g + 1];
  const int nl = l1 - l0, n = nl + (p1 - p0);
  float sx = 0.f, sy = 0.f, sz = 0.f;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    const int i = k < nl ? l0 + k : p0 + (k - nl);
    const float4 a = x_fin[i], b = x_in[i];
    sx += a.x - b.x; sy += a.y - b.y; sz += a.z - b.z;
  }
  __shared__ float red[3][4];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sx += __shfl_xor_sync(0xffffffffu, sx, o);
    sy += __shfl_xor_sync(0xffffffffu, sy, o);
    sz += __shfl_xor_sync(0xffffffffu, sz, o);
  }
  const int wid = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { red[0][wid] = sx; red[1][wid] = sy; red[2][wid] = sz; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const float cnt = n > 0 ? (float)n : 1.f;
    velmean[g] = make_float4((red[0][0] + red[0][1] + red[0][2] + red[0][3]) / cnt,
                             (red[1][0] + red[1][1] + red[1][2] + red[1][3]) / cnt,
                             (red[2][0] + red[2][1] + red[2][2] + red[2][3]) / cnt, 0.f);
  }
}

// embedding_out (H -> J+1, time channel dropped, egnn_new.py:241 / dynamics.py:149) and the decoder's first Linear
// are folded at pack time into one [2F][H] matrix per node type; a warp owns 4 nodes: lanes split the H axis of
// the fused first layer (butterfly reduction), the tiny second Linear runs from a per-warp shared buffer.
constexpr int POST_WARPS = PREP_THREADS / 32;
constexpr int POST_NPW = PREP_NODES / POST_WARPS;      // nodes per warp (4)
constexpr int POST_MAX_F2 = 128;

struct PostArgs {
  const float* h; const float4* x_fin; const float4* x_in; const int32_t* gid; const float4* velmean;
  int NL, NP, A, R, H; int joint;
  const float *dec_w[2], *dec_b[2];
  const float *adec2_w, *adec2_b, *rdec2_w, *rdec2_b;
  float* out_atoms; float* out_res; int32_t* status;
};

__global__ void __launch_bounds__(PREP_THREADS) post_kernel(PostArgs p) {
  pdl_trigger();
  pdl_wait();
  __shared__ float s_hid[POST_WARPS][POST_NPW][POST_MAX_F2];
  const int lig_blocks = (p.NL + PREP_NODES - 1) / PREP_NODES;
  const bool is_lig = blockIdx.x < lig_blocks;
  const int F = is_lig ? p.A : p.R, F2 = 2 * F;
  const int base = is_lig ? blockIdx.x * PREP_NODES : (blockIdx.x - lig_blocks) * PREP_NODES;
  const int count = is_lig ? p.NL : p.NP;
  const int nn = min(PREP_NODES, count - base);
  const int node0 = is_lig ? base : p.NL + base;
  float* out = is_lig ? p.out_atoms : p.out_res;
  const int ld = 3 + F;
  const float* w1 = p.dec_w[is_lig ? 0 : 1];
  const float* b1 = p.dec_b[is_lig ? 0 : 1];
  const float *w2 = is_lig ? p.adec2_w : p.rdec2_w, *b2 = is_lig ? p.adec2_b : p.rdec2_b;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid < nn) {
    const float4 a = p.x_fin[node0 + tid], b = p.x_in[node0 + tid];
    float vx = a.x - b.x, vy = a.y - b.y, vz = a.z - b.z;
    if (isnan(vx) || isnan(vy) || isnan(vz)) atomicOr(&p.status[0], 1);   // dynamics.py:155-159
    if (p.joint) {                                                         // dynamics.py:161-164
      const float4 m = p.velmean[p.gid[node0 + tid]];
      vx -= m.x; vy -= m.y; vz -= m.z;
    }
    float* row = out + (size_t)(base + tid) * ld;
    row[0] = vx; row[1] = vy; row[2] = vz;
  }

  const int nl0 = warp * POST_NPW;                  // first local node of this warp
  if (nl0 >= nn) return;
  const int H4 = p.H >> 2;
  float4 hv[POST_NPW][2];
#pragma unroll
  for (int j = 0; j < POST_NPW; ++j)
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int k4 = lane + 32 * q;
      hv[j][q] = (nl0 + j < nn && k4 < H4)
                     ? *reinterpret_cast<const float4*>(p.h + (size_t)(node0 + nl0 + j) * p.H + 4 * k4)
                     : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  for (int o = 0; o < F2; ++o) {
    float acc[POST_NPW];
#pragma unroll
    for (int j = 0; j < POST_NPW; ++j) acc[j] = 0.f;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int k4 = lane + 32 * q;
      if (k4 < H4) {
        const float4 w = __ldg(reinterpret_cast<const float4*>(w1 + (size_t)o * p.H) + k4);
#pragma unroll
        for (int j = 0; j < POST_NPW; ++j)
          acc[j] = fmaf(w.x, hv[j][q].x, fmaf(w.y, hv[j][q].y, fmaf(w.z, hv[j][q].z, fmaf(w.w, hv[j][q].w, acc[j]))));
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
#pragma unroll
      for (int j = 0; j < POST_NPW; ++j) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], off);
    if (lane < POST_NPW) {
      const float v = lane == 0 ? acc[0] : lane == 1 ? acc[1] : lane == 2 ? acc[2] : acc[3];
      s_hid[warp][lane][o] = silu_f(v + b1[o]);
    }
  }
  __syncwarp();
  for (int i = lane; i < POST_NPW * F; i += 32) {
    const int j = i / F, o = i - j * F;
    if (nl0 + j >= nn) continue;
    float acc = b2[o];
    for (int k = 0; k < F2; ++k) acc = fmaf(s_hid[warp][j][k], w2[o * F2 + k], acc);
    out[(size_t)(base + nl0 + j) * ld + 3 + o] = acc;
  }
}

int launch_post(const dsb_dynamics* d, const Dims& dm, const Workspace& ws, const float4* x_final,
                float* out_atoms, float* out_residues, int32_t* status, cudaStream_t s, int max_launches) {
  const dsb_config& c = d->cfg;
  const PackedWeights& w = d->w;
  static_assert(POST_NPW == 4, "lane select below assumes 4 nodes per warp");
  if (c.update_pocket_coords && dm.B > 0) {
    if (max_launches < 1) return 0;
    DSB_CUDA_OK(launch_k(velmean_kernel, dm.B, 128, 0, s, x_final, ws.xbuf[0], ws.lig_off, ws.poc_off, dm.NL, ws.velmean));
    --max_launches;
  }
  if (max_launches < 1) return 0;
  PostArgs p;
  p.h = ws.h; p.x_fin = x_final; p.x_in = ws.xbuf[0]; p.gid = ws.gid; p.velmean = ws.velmean;
  p.NL = dm.NL; p.NP = dm.NP; p.A = c.atom_nf; p.R = c.residue_nf; p.H = c.hidden_nf; p.joint = c.update_pocket_coords;
  p.dec_w[0] = w.dec_w[0]; p.dec_w[1] = w.dec_w[1]; p.dec_b[0] = w.dec_b[0]; p.dec_b[1] = w.dec_b[1];
  p.adec2_w = w.adec2_w; p.adec2_b = w.adec2_b; p.rdec2_w = w.rdec2_w; p.rdec2_b = w.rdec2_b;
  p.out_atoms = out_atoms; p.out_res = out_residues; p.status = status;
  int blocks = (dm.NL + PREP_NODES - 1) / PREP_NODES + (dm.NP + PREP_NODES - 1) / PREP_NODES;
  if (blocks == 0) return 0;
  DSB_CUDA_OK(launch_k(post_kernel, blocks, PREP_THREADS, 0, s, p));
  return 0;
}

// =====================================================================================================
// node GEMM: C[M][Nn] = act( [A1 | A2/div2] @ W + bias ) (+ R).  fp32 SIMT, 128x128x16 tiles, 256 threads,
// 8x8 register micro-tiles, register-staged double buffering.  Used for the factorised first layers of
// the edge/coord MLPs (W1a*h_i, W1b*h_j), node_mlp (egnn_new.py:21-24, :56-57).
// =====================================================================================================
constexpr int GBM = 128, GBN = 128, GBK = 16, GTHREADS = 256;

__global__ void __launch_bounds__(GTHREADS, 2) node_gemm_kernel(GemmArgs g) {
  __shared__ __align__(16) float As[2][GBK][GBM + 4];
  __shared__ __align__(16) float Bs[2][GBK][GBN];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * GBM, n0 = blockIdx.x * GBN;
  if (g.dead_cols > 0 && m0 >= g.dead_rows_from && n0 + GBN <= g.dead_cols) return;   // whole tile is in the unused block
  const int K = g.K1 + g.K2;
  const int tx = tid & 15, ty = tid >> 4;

  // loader mapping: A tile 128 rows x 16 k = 512 float4 -> 2 per thread; B tile 16 k x 128 n = 512 float4
  const int a_r = tid >> 2;            // 0..63 (+64)
  const int a_k4 = (tid & 3) * 4;      // 0,4,8,12
  const int b_k = tid >> 5;            // 0..7 (+8)
  const int b_n4 = (tid & 31) * 4;     // 0..124

  float4 ra[2], rb[2];
  auto load_tiles = [&](int k0) {
    const bool second = k0 >= g.K1;
    const float* A = second ? g.A2 : g.A1;
    const int lda = second ? g.lda2 : g.lda1;
    const int kk = second ? k0 - g.K1 : k0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int m = m0 + a_r + 64 * i;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m < g.M) {
        v = *reinterpret_cast<const float4*>(A + (size_t)m * lda + kk + a_k4);
        if (second && (g.div2 != 1.0f || g.deg2)) {
          const float dv = g.deg2 ? (float)max(g.deg2[m], 1) : g.div2;      // 'mean': the receiver's edge count (egnn_new.py:330-334)
          v.x = __fdiv_rn(v.x, dv); v.y = __fdiv_rn(v.y, dv);
          v.z = __fdiv_rn(v.z, dv); v.w = __fdiv_rn(v.w, dv);
        }
      }
      ra[i] = v;
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int k = k0 + b_k + 8 * i;
      const int n = n0 + b_n4;
      rb[i] = (n < g.Nn) ? *reinterpret_cast<const float4*>(g.W + (size_t)k * g.ldw + n)
                         : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = a_r + 64 * i;
      As[buf][a_k4 + 0][r] = ra[i].x; As[buf][a_k4 + 1][r] = ra[i].y;
      As[buf][a_k4 + 2][r] = ra[i].z; As[buf][a_k4 + 3][r] = ra[i].w;
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) *reinterpret_cast<float4*>(&Bs[buf][b_k + 8 * i][b_n4]) = rb[i];
  };

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  int buf = 0;
  for (int k0 = 0; k0 < K; k0 += GBK) {
    const bool nxt = k0 + GBK < K;
    if (nxt) load_tiles(k0 + GBK);
#pragma unroll
    for (int kk = 0; kk < GBK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (nxt) store_tiles(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }

  // epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= g.M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int n = n0 + jh * 64 + tx * 4;
      if (n >= g.Nn) continue;
      float v[4] = {acc[i][jh * 4 + 0], acc[i][jh * 4 + 1], acc[i][jh * 4 + 2], acc[i][jh * 4 + 3]};
      if (g.bias) {
        const float4 b = *reinterpret_cast<const float4*>(g.bias + n);
        v[0] += b.x; v[1] += b.y; v[2] += b.z; v[3] += b.w;
      }
      if (g.act == 1) {
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = silu_f(v[q]);
      }
      if (g.R) {
        const float4 r = *reinterpret_cast<const float4*>(g.R + (size_t)m * g.ldr + n);
        v[0] = r.x + v[0]; v[1] = r.y + v[1]; v[2] = r.z + v[2]; v[3] = r.w + v[3];
      }
      *reinterpret_cast<float4*>(g.C + (size_t)m * g.ldc + n) = make_float4(v[0], v[1], v[2], v[3]);
      if (g.Z) *reinterpret_cast<float4*>(g.Z + (size_t)m * g.ldz + n) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// All kernels of the library ask for the maximum shared-memory carve-out: the tensor-core kernels need ~225 KB, and an SM
// that has to switch its L1/shared split between consecutive launches drains first.  The small kernels do not depend on L1.
int configure_node_kernels() {
  const int mx = cudaSharedmemCarveoutMaxShared;
  DSB_CUDA_OK(cudaFuncSetAttribute(plan_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
  DSB_CUDA_OK(cudaFuncSetAttribute(prep_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
  DSB_CUDA_OK(cudaFuncSetAttribute(edge_rows_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
  DSB_CUDA_OK(cudaFuncSetAttribute(edge_rows_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
  DSB_CUDA_OK(cudaFuncSetAttribute(scan_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
  DSB_CUDA_OK(cudaFuncSetAttribute(coord_finish_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
  DSB_CUDA_OK(cudaFuncSetAttribute(velmean_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
  DSB_CUDA_OK(cudaFuncSetAttribute(post_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
  DSB_CUDA_OK(cudaFuncSetAttribute(node_gemm_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, mx));
  return 0;
}

int launch_node_gemm(const GemmArgs& a, cudaStream_t s) {
  if (a.M == 0) return 0;
  if ((a.K1 % GBK) || (a.K2 % GBK) || (a.Nn % 4) || (a.ldw % 4) || (a.ldc % 4) || (a.lda1 % 4)) {
    set_error("node_gemm: unsupported shape K1=%d K2=%d Nn=%d", a.K1, a.K2, a.Nn);
    return DSB_ERR_INVALID_ARGUMENT;
  }
  dim3 grid((a.Nn + GBN - 1) / GBN, (a.M + GBM - 1) / GBM);
  node_gemm_kernel<<<grid, GTHREADS, 0, s>>>(a);
  DSB_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace dsb
