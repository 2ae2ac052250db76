// Edge-level kernels: the O(E * H^2) part of the denoiser (99 % of the FLOPs, SURVEY.md §8(a) rows a8/a10).
//
//   edge_gcl_kernel   — GCL.edge_model + receiver-side segment sum   (egnn_new.py:31-52)
//   edge_coord_kernel — EquivariantUpdate.coord_model                 (egnn_new.py:96-116)
//
// Both are persistent kernels (one CTA per SM) over tiles of 128 consecutive CSR edges (edges are sorted
// by receiver row, so a tile covers a few whole receivers plus at most two partial ones).  Per tile:
//   1. per-edge scalars (row, col, d^2 of the current geometry, d^2 of the input geometry, edge type,
//      and for the coordinate kernel the normalised difference / cross-product directions) -> shared memory
//   2. first layer, factorised:  X[e][k] = SiLU( Pa[row_e][k] + Pb[col_e][k] + d2_e*wr[k] + d0_e*wr0[k] (+ tb[type_e][k]) )
//      where Pa = W1a*h_i + b1 and Pb = W1b*h_j were produced by the node GEMM — built chunk-wise (32 k at a
//      time) straight into shared memory, never materialised in HBM (the reference materialises [E, 2H+2] thrice per block)
//   3. second layer: acc[128][H] += X_chunk @ W2_chunk, fp32 FFMA, 8 x (H/16) register micro-tile per thread,
//      W2 chunks streamed from L2 with cp.async double buffering
//   4. epilogue in registers: +b2, SiLU, attention gate (half-warp shuffle reduce) or phi = w3 . m
//   5. deterministic-order segmented sum over the tile's rows through shared memory; one RED per
//      (receiver segment, column) into the zero-initialised aggregate — no per-edge atomics.
// DET (deterministic mode): the tiles run over the padded virtual edge order of the tensor-core kernels (vrow_ptr / vmap:
// every receiver starts at a multiple of kRowChunk rows), step 5 stores the in-order sum of every 4-row chunk into the
// chunk's slot of Workspace::part, and launch_segment_reduce sums each receiver's chunks in ascending order.  A receiver's
// sum then depends on its own edges only, not on where the 128-edge tiles fall or on the order the tiles finish.
#include "dsb_internal.cuh"

namespace dsb {

constexpr int EBM = 128;     // edges per tile
constexpr int EKC = 32;      // k-chunk
constexpr int ETHREADS = 256;
constexpr int EXS = EBM + 4; // padded row stride of the k-major X chunk

template <int H>
struct EdgeSmem {
  static constexpr int NQ = H / 64;
  static constexpr int kXs = 2 * EKC * EXS;          // floats
  static constexpr int kWs = 2 * EKC * H;            // floats
  static constexpr int kMain = kXs + kWs;            // floats, reused as the epilogue tile
  static constexpr int kEs = EBM * (128 + 4);        // floats needed by the segmented reduce
  static constexpr int kMainAlloc = kMain > kEs ? kMain : kEs;
};

// ---- shared main loop --------------------------------------------------------------------------------
// acc[i][q*4+j] accumulates row (ty*8+i), column (64*q + tx*4 + j) of  X @ W2.
template <int H, bool SIN>
__device__ __forceinline__ void edge_mlp_mainloop(
    float (&acc)[8][H / 16], float* __restrict__ Xs, float* __restrict__ Ws,
    const float* __restrict__ P, int ldp, int offA, int offB,
    const float* __restrict__ s_wr, const float* __restrict__ s_wr0, const float* __restrict__ s_tb,
    const int* __restrict__ s_row, const int* __restrict__ s_col, const float* __restrict__ s_d2,
    const float* __restrict__ s_d0, const int* __restrict__ s_type,
    const float* __restrict__ W2,
    const float* __restrict__ g_wr = nullptr, const float* __restrict__ g_wr0 = nullptr) {
  // g_wr != nullptr: sin_embedding (egnn_new.py:282-293).  The two distances enter the first layer as 12 sinusoids each:
  // [sin(f_k d) | cos(f_k d)], f_k = 2 pi 4^k / 15, d = sqrt(d^2 + 1e-8); g_wr / g_wr0 = their [12][H] weight rows (global
  // memory, L1-resident).  24 FMAs per first-layer value instead of 2: the flag is unused by every shipped config and is
  // built for completeness, not speed.
  constexpr int NQ = H / 64;
  constexpr int NCH = H / EKC;
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  // X producer mapping: edge row r, alternating k-quads (conflict-free transposed stores)
  const int pr = tid >> 1, phf = tid & 1;
  const int prow = s_row[pr] < 0 ? 0 : s_row[pr];
  const int pcol = s_col[pr];
  const float pd2 = s_d2[pr], pd0 = s_d0[pr];
  const int ptype = s_type ? s_type[pr] : 0;
  float emb[SIN ? 24 : 1];
  if constexpr (SIN) {
    const float dc = sqrtf(pd2 + 1e-8f), di = sqrtf(pd0 + 1e-8f);
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const float f = __fdiv_rn(6.2831853071795864769f * (float)(1 << (2 * k)), 15.0f);      // torch: fp32(2 pi) * 4^k / 15
      emb[k] = sinf(dc * f); emb[6 + k] = cosf(dc * f);
      emb[12 + k] = sinf(di * f); emb[18 + k] = cosf(di * f);
    }
  }
  const float* Pa = P + (size_t)prow * ldp + offA;
  const float* Pb = P + (size_t)pcol * ldp + offB;

#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < H / 16; ++j) acc[i][j] = 0.f;

  float4 ga[4], gb[4];
  auto x_load = [&](int kc) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int k0 = kc * EKC + (phf + 2 * q) * 4;
      ga[q] = *reinterpret_cast<const float4*>(Pa + k0);
      gb[q] = *reinterpret_cast<const float4*>(Pb + k0);
    }
  };
  auto x_store = [&](int kc, int buf) {
    float* X = Xs + buf * (EKC * EXS);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int kl = (phf + 2 * q) * 4;
      const int k0 = kc * EKC + kl;
      float v[4] = {ga[q].x + gb[q].x, ga[q].y + gb[q].y, ga[q].z + gb[q].z, ga[q].w + gb[q].w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float u;
        if constexpr (SIN) {
          u = v[j];
#pragma unroll
          for (int f = 0; f < 12; ++f) u = fmaf(emb[f], __ldg(g_wr + f * H + k0 + j), u);
#pragma unroll
          for (int f = 0; f < 12; ++f) u = fmaf(emb[12 + f], __ldg(g_wr0 + f * H + k0 + j), u);
        } else {
          u = fmaf(pd2, s_wr[k0 + j], v[j]);
          u = fmaf(pd0, s_wr0[k0 + j], u);
        }
        if (s_tb) u += s_tb[ptype * H + k0 + j];
        X[(kl + j) * EXS + pr] = silu_f(u);
      }
    }
  };
  auto w_issue = [&](int kc, int buf) {
    float* W = Ws + buf * (EKC * H);
    const float* src = W2 + (size_t)kc * EKC * H;
#pragma unroll
    for (int i = 0; i < (EKC * H / 4) / ETHREADS; ++i) {
      const int idx = tid + ETHREADS * i;
      cp_async16(W + idx * 4, src + idx * 4);
    }
    cp_async_commit();
  };

  w_issue(0, 0);
  x_load(0);
  x_store(0, 0);
  cp_async_wait_all();
  __syncthreads();

  int buf = 0;
#pragma unroll 1
  for (int kc = 0; kc < NCH; ++kc) {
    const bool nxt = kc + 1 < NCH;
    if (nxt) { w_issue(kc + 1, buf ^ 1); x_load(kc + 1); }
    const float* X = Xs + buf * (EKC * EXS) + ty * 8;
    const float* W = Ws + buf * (EKC * H) + tx * 4;
#pragma unroll 8
    for (int kk = 0; kk < EKC; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(X + kk * EXS);
      const float4 a1 = *reinterpret_cast<const float4*>(X + kk * EXS + 4);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const float4 b = *reinterpret_cast<const float4*>(W + kk * H + 64 * q);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          acc[i][q * 4 + 0] = fmaf(av[i], b.x, acc[i][q * 4 + 0]);
          acc[i][q * 4 + 1] = fmaf(av[i], b.y, acc[i][q * 4 + 1]);
          acc[i][q * 4 + 2] = fmaf(av[i], b.z, acc[i][q * 4 + 2]);
          acc[i][q * 4 + 3] = fmaf(av[i], b.w, acc[i][q * 4 + 3]);
        }
      }
    }
    if (nxt) { x_store(kc + 1, buf ^ 1); cp_async_wait_all(); }
    __syncthreads();
    buf ^= 1;
  }
}

// =====================================================================================================
struct EdgeGclArgs {
  const float* P; int ldp;           // [N][2H]: cols 0..H-1 = W1a*h+b1, H..2H-1 = W1b*h
  const float4* x;                   // current coordinates
  const int32_t* row_ptr; int N;     // E = row_ptr[N]
  const int32_t *erow, *ecol; const float* ed0; int NL;
  GclW w;
  float* agg;                        // [N][H], zero on entry; receives raw sums
  const int32_t* vrow_ptr; const int32_t* vmap; float* part;   // DET: virtual rows, chunk partials [chunk][H]
  int vcap;                                                     // DET: virtual rows covered by vmap / part
};

template <int H, bool SIN, bool DET = false>
__global__ void __launch_bounds__(ETHREADS, 1) edge_gcl_kernel(EdgeGclArgs a) {
  extern __shared__ __align__(16) float smem[];
  using S = EdgeSmem<H>;
  constexpr int NQ = H / 64;
  float* Xs = smem;
  float* Ws = smem + S::kXs;
  float* s_wr = smem + S::kMainAlloc;
  float* s_wr0 = s_wr + H;
  float* s_b2 = s_wr0 + H;
  float* s_wa = s_b2 + H;
  float* s_tb = s_wa + H;                       // [3][H]
  float* s_d2 = s_tb + 3 * H;
  float* s_d0 = s_d2 + EBM;
  int* s_row = reinterpret_cast<int*>(s_d0 + EBM);
  int* s_col = s_row + EBM;
  int* s_type = s_col + EBM;

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const bool has_tb = a.w.tb != nullptr, has_att = a.w.wa != nullptr;
  for (int i = tid; i < H; i += ETHREADS) {
    s_wr[i] = a.w.wr[i]; s_wr0[i] = a.w.wr0[i]; s_b2[i] = a.w.b2[i];
    s_wa[i] = has_att ? a.w.wa[i] : 0.f;
    if (has_tb) { s_tb[i] = a.w.tb[i]; s_tb[H + i] = a.w.tb[H + i]; s_tb[2 * H + i] = a.w.tb[2 * H + i]; }
  }
  const float ba = has_att ? a.w.ba[0] : 0.f;
  const int E = DET ? min(a.vrow_ptr[a.N], a.vcap) : a.row_ptr[a.N];
  __syncthreads();

#pragma unroll 1
  for (int e0 = blockIdx.x * EBM; e0 < E; e0 += gridDim.x * EBM) {
    if (tid < EBM) {
      const int e = DET ? (e0 + tid < E ? a.vmap[e0 + tid] : -1) : e0 + tid;
      int r = -1, c = 0, ty_ = 0; float d2 = 0.f, d0 = 0.f;
      if (DET ? e >= 0 : e < E) {
        r = a.erow[e]; c = a.ecol[e]; d0 = a.ed0[e];
        const float4 xi = a.x[r], xj = a.x[c];
        const float dx = xi.x - xj.x, dy = xi.y - xj.y, dz = xi.z - xj.z;
        d2 = dx * dx + dy * dy + dz * dz;
        ty_ = (r < a.NL) == (c < a.NL) ? (r < a.NL ? 1 : 2) : 0;   // dynamics.py:119-122
      }
      s_row[tid] = r; s_col[tid] = c; s_d2[tid] = d2; s_d0[tid] = d0; s_type[tid] = ty_;
    }
    __syncthreads();

    float acc[8][H / 16];
    edge_mlp_mainloop<H, SIN>(acc, Xs, Ws, a.P, a.ldp, 0, H, s_wr, s_wr0, has_tb ? s_tb : nullptr,
                              s_row, s_col, s_d2, s_d0, has_tb ? s_type : nullptr, a.w.W2, a.w.wr, a.w.wr0);

    // ---- epilogue: m = SiLU(acc + b2); e = m * sigmoid(wa.m + ba)  (egnn_new.py:36-40)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float s = 0.f;
#pragma unroll
      for (int q = 0; q < NQ; ++q)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = 64 * q + tx * 4 + j;
          const float m = silu_f(acc[i][q * 4 + j] + s_b2[c]);
          acc[i][q * 4 + j] = m;
          s = fmaf(m, s_wa[c], s);
        }
      if (has_att) {
        s += __shfl_xor_sync(0xffffffffu, s, 8);
        s += __shfl_xor_sync(0xffffffffu, s, 4);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        const float g = sigmoid_f(s + ba);
#pragma unroll
        for (int j = 0; j < H / 16; ++j) acc[i][j] *= g;
      }
    }

    // ---- segmented sum over the tile's edge rows, 128 columns per pass (egnn_new.py:50-52, :326)
    float* Es = smem;    // [EBM][132], aliases the main-loop buffers (all reads finished at the loop's last barrier)
    constexpr int NPASS = (H + 127) / 128;
#pragma unroll
    for (int pass = 0; pass < NPASS; ++pass) {
#pragma unroll
      for (int q = 2 * pass; q < 2 * pass + 2 && q < NQ; ++q)
#pragma unroll
        for (int i = 0; i < 8; ++i)
          *reinterpret_cast<float4*>(Es + (ty * 8 + i) * 132 + (q - 2 * pass) * 64 + tx * 4) =
              make_float4(acc[i][q * 4 + 0], acc[i][q * 4 + 1], acc[i][q * 4 + 2], acc[i][q * 4 + 3]);
      __syncthreads();
      const int c = tid & 127, rh = tid >> 7;
      const int ncols = (H - 128 * pass) < 128 ? (H - 128 * pass) : 128;
      if constexpr (DET) {
        if (c < ncols) {
          constexpr int NCH = EBM / kRowChunk;
          for (int k = rh * (NCH / 2); k < (rh + 1) * (NCH / 2); ++k) {
            float sum = 0.f;
#pragma unroll
            for (int i = 0; i < kRowChunk; ++i) {
              const int r = k * kRowChunk + i;
              if (s_row[r] >= 0) sum += Es[r * 132 + c];
            }
            a.part[(size_t)(e0 / kRowChunk + k) * H + 128 * pass + c] = sum;
          }
        }
      } else if (c < ncols) {
        int cur = -1; float sum = 0.f;
        for (int r = rh * 64; r < rh * 64 + 64; ++r) {
          const int row = s_row[r];
          if (row != cur) {
            if (cur >= 0) atomicAdd(a.agg + (size_t)cur * H + 128 * pass + c, sum);
            cur = row; sum = 0.f;
          }
          if (row >= 0) sum += Es[r * 132 + c];
        }
        if (cur >= 0) atomicAdd(a.agg + (size_t)cur * H + 128 * pass + c, sum);
      }
      __syncthreads();
    }
  }
}

// =====================================================================================================
struct EdgeCoordArgs {
  const float* P; int ldp;           // [N][nm*2H]: receiver block (m*H) then sender block (nm*H + m*H)
  const float4* x; const float4* cent; const int32_t* gid;
  const int32_t* row_ptr; int n_rows;   // edges [0, row_ptr[n_rows]) have a moving receiver
  const int32_t *erow, *ecol; const float* ed0; int NL;
  EquivW w; int nm;                  // nm = 1 (reflection equivariant) or 2 (+ cross-product MLP)
  float norm_constant, coords_range; int use_tanh;
  float4* xagg;                      // [N], zero on entry; receives raw sums of trans
  const int32_t* vrow_ptr; const int32_t* vmap; float4* part;  // DET: virtual rows, chunk partials [chunk] (both MLPs summed)
  int vcap;                                                     // DET: virtual rows covered by vmap / part
};

template <int H, bool SIN, bool DET = false>
__global__ void __launch_bounds__(ETHREADS, 1) edge_coord_kernel(EdgeCoordArgs a) {
  extern __shared__ __align__(16) float smem[];
  using S = EdgeSmem<H>;
  constexpr int NQ = H / 64;
  float* Xs = smem;
  float* Ws = smem + S::kXs;
  float* s_vec = smem + S::kMainAlloc;          // per MLP m: wr, wr0, b2, tb[3]  -> 6H each; then w3
  float* s_w3 = s_vec + 2 * 6 * H;
  float* s_d2 = s_w3 + H;
  float* s_d0 = s_d2 + EBM;
  float* s_phi = s_d0 + EBM;                    // [2][EBM]
  float* s_dir = s_phi + 2 * EBM;               // [6][EBM]: diff xyz, cross xyz
  int* s_row = reinterpret_cast<int*>(s_dir + 6 * EBM);
  int* s_col = s_row + EBM;
  int* s_type = s_col + EBM;

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const bool has_tb = a.w.tb[0] != nullptr;
  for (int i = tid; i < H; i += ETHREADS) {
    for (int m = 0; m < a.nm; ++m) {
      float* v = s_vec + m * 6 * H;
      v[i] = a.w.wr[m][i]; v[H + i] = a.w.wr0[m][i]; v[2 * H + i] = a.w.b2[m][i];
      if (has_tb) { v[3 * H + i] = a.w.tb[m][i]; v[4 * H + i] = a.w.tb[m][H + i]; v[5 * H + i] = a.w.tb[m][2 * H + i]; }
    }
    s_w3[i] = a.w.w3[i];
  }
  const int E = DET ? min(a.vrow_ptr[a.n_rows], a.vcap) : a.row_ptr[a.n_rows];
  __syncthreads();

#pragma unroll 1
  for (int e0 = blockIdx.x * EBM; e0 < E; e0 += gridDim.x * EBM) {
    if (tid < EBM) {
      const int e = DET ? (e0 + tid < E ? a.vmap[e0 + tid] : -1) : e0 + tid;
      int r = -1, c = 0, ty_ = 0; float d2 = 0.f, d0 = 0.f;
      float dir[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (DET ? e >= 0 : e < E) {
        r = a.erow[e]; c = a.ecol[e]; d0 = a.ed0[e];
        const float4 xi = a.x[r], xj = a.x[c];
        const float dx = xi.x - xj.x, dy = xi.y - xj.y, dz = xi.z - xj.z;
        d2 = dx * dx + dy * dy + dz * dz;
        ty_ = (r < a.NL) == (c < a.NL) ? (r < a.NL ? 1 : 2) : 0;
        const float den = sqrtf(d2 + 1e-8f) + a.norm_constant;           // egnn_new.py:300-301
        dir[0] = dx / den; dir[1] = dy / den; dir[2] = dz / den;
        if (a.nm == 2) {                                                  // egnn_new.py:312-315
          const float4 m = a.cent[a.gid[r]];
          const float ax = xi.x - m.x, ay = xi.y - m.y, az = xi.z - m.z;
          const float bx = xj.x - m.x, by = xj.y - m.y, bz = xj.z - m.z;
          const float cx = ay * bz - az * by, cy = az * bx - ax * bz, cz = ax * by - ay * bx;
          const float cn = sqrtf(cx * cx + cy * cy + cz * cz) + a.norm_constant;
          dir[3] = cx / cn; dir[4] = cy / cn; dir[5] = cz / cn;
        }
      }
      s_row[tid] = r; s_col[tid] = c; s_d2[tid] = d2; s_d0[tid] = d0; s_type[tid] = ty_;
#pragma unroll
      for (int k = 0; k < 6; ++k) s_dir[k * EBM + tid] = dir[k];
    }
    __syncthreads();

#pragma unroll 1
    for (int m = 0; m < a.nm; ++m) {
      float acc[8][H / 16];
      const float* v = s_vec + m * 6 * H;
      edge_mlp_mainloop<H, SIN>(acc, Xs, Ws, a.P, a.ldp, m * H, a.nm * H + m * H, v, v + H,
                                has_tb ? v + 3 * H : nullptr, s_row, s_col, s_d2, s_d0,
                                has_tb ? s_type : nullptr, a.w.W2[m], a.w.wr[m], a.w.wr0[m]);
      const float* b2 = v + 2 * H;
#pragma unroll
      for (int i = 0; i < 8; ++i) {   // phi = w3 . SiLU(acc + b2)   (egnn_new.py:83-85, bias-free last layer)
        float s = 0.f;
#pragma unroll
        for (int q = 0; q < NQ; ++q)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = 64 * q + tx * 4 + j;
            s = fmaf(silu_f(acc[i][q * 4 + j] + b2[c]), s_w3[c], s);
          }
        s += __shfl_xor_sync(0xffffffffu, s, 8);
        s += __shfl_xor_sync(0xffffffffu, s, 4);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        if (tx == 0) s_phi[m * EBM + ty * 8 + i] = s;
      }
    }
    __syncthreads();
    // trans = dir * tanh(phi) * range (+ cross * tanh(phi_x) * range)   (egnn_new.py:100-109)
    float* s_tr = Xs;   // [3][EBM], main-loop buffers are idle here
    if (tid < EBM) {
      float p0 = s_phi[tid];
      float t0, t1 = 0.f;
      if (a.use_tanh) { t0 = tanhf(p0) * a.coords_range; } else { t0 = p0; }
      if (a.nm == 2) { const float p1 = s_phi[EBM + tid]; t1 = a.use_tanh ? tanhf(p1) * a.coords_range : p1; }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        float tr = a.use_tanh ? (s_dir[k * EBM + tid] * tanhf(p0)) * a.coords_range : s_dir[k * EBM + tid] * t0;
        if (a.nm == 2) tr = tr + s_dir[(3 + k) * EBM + tid] * t1;
        s_tr[k * EBM + tid] = tr;
      }
    }
    __syncthreads();
    if constexpr (DET) {
      if (tid < EBM / kRowChunk) {      // in-order 4-row chunk sums -> the chunk's slot
        float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int i = 0; i < kRowChunk; ++i) {
          const int r = tid * kRowChunk + i;
          if (s_row[r] >= 0) { sum.x += s_tr[r]; sum.y += s_tr[EBM + r]; sum.z += s_tr[2 * EBM + r]; }
        }
        a.part[e0 / kRowChunk + tid] = sum;
      }
    } else if (tid < 3) {      // in-order segmented sum (egnn_new.py:114-116)
      int cur = -1; float sum = 0.f;
      float* dst = reinterpret_cast<float*>(a.xagg);
      for (int r = 0; r < EBM; ++r) {
        const int row = s_row[r];
        if (row != cur) {
          if (cur >= 0) atomicAdd(dst + (size_t)cur * 4 + tid, sum);
          cur = row; sum = 0.f;
        }
        if (row >= 0) sum += s_tr[tid * EBM + r];
      }
      if (cur >= 0) atomicAdd(dst + (size_t)cur * 4 + tid, sum);
    }
    __syncthreads();
  }
}

// =====================================================================================================
template <int H> static size_t gcl_smem_bytes() {
  return sizeof(float) * (size_t)(EdgeSmem<H>::kMainAlloc + 7 * H + 2 * EBM) + sizeof(int) * 3 * EBM;
}
template <int H> static size_t coord_smem_bytes() {
  return sizeof(float) * (size_t)(EdgeSmem<H>::kMainAlloc + 13 * H + 10 * EBM) + sizeof(int) * 3 * EBM;
}

template <int H, bool DET> static int configure_variant() {
  DSB_CUDA_OK(cudaFuncSetAttribute(edge_gcl_kernel<H, false, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gcl_smem_bytes<H>()));
  DSB_CUDA_OK(cudaFuncSetAttribute(edge_coord_kernel<H, false, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)coord_smem_bytes<H>()));
  DSB_CUDA_OK(cudaFuncSetAttribute(edge_gcl_kernel<H, true, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gcl_smem_bytes<H>()));
  DSB_CUDA_OK(cudaFuncSetAttribute(edge_coord_kernel<H, true, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)coord_smem_bytes<H>()));
  return 0;
}
template <int H> static int configure_h() {
  if (int e = configure_variant<H, false>()) return e;
  return configure_variant<H, true>();
}

template <int H> static void run_gcl(const EdgeGclArgs& a, bool sin, bool det, int grid, cudaStream_t s) {
  const size_t sm = gcl_smem_bytes<H>();
  if (det) { if (sin) edge_gcl_kernel<H, true, true><<<grid, ETHREADS, sm, s>>>(a); else edge_gcl_kernel<H, false, true><<<grid, ETHREADS, sm, s>>>(a); }
  else { if (sin) edge_gcl_kernel<H, true><<<grid, ETHREADS, sm, s>>>(a); else edge_gcl_kernel<H, false><<<grid, ETHREADS, sm, s>>>(a); }
}
template <int H> static void run_coord(const EdgeCoordArgs& a, bool sin, bool det, int grid, cudaStream_t s) {
  const size_t sm = coord_smem_bytes<H>();
  if (det) { if (sin) edge_coord_kernel<H, true, true><<<grid, ETHREADS, sm, s>>>(a); else edge_coord_kernel<H, false, true><<<grid, ETHREADS, sm, s>>>(a); }
  else { if (sin) edge_coord_kernel<H, true><<<grid, ETHREADS, sm, s>>>(a); else edge_coord_kernel<H, false><<<grid, ETHREADS, sm, s>>>(a); }
}

int configure_edge_kernels(int H) {
  switch (H) {
    case 64: return configure_h<64>();
    case 128: return configure_h<128>();
    case 192: return configure_h<192>();
    case 256: return configure_h<256>();
    default: set_error("hidden_nf=%d unsupported (64,128,192,256)", H); return DSB_ERR_UNSUPPORTED_CONFIG;
  }
}

int launch_edge_gcl(const dsb_dynamics* d, const Dims& dm, const Workspace& ws, const GclW& w,
                    const float4* x, PView pv, cudaStream_t s) {
  const int H = d->cfg.hidden_nf;
  EdgeGclArgs a;
  a.P = pv.P; a.ldp = pv.ldp; a.x = x; a.row_ptr = ws.row_ptr; a.N = dm.N;
  a.erow = ws.erow; a.ecol = ws.ecol; a.ed0 = ws.ed0; a.NL = dm.NL; a.w = w; a.agg = ws.agg;
  a.vrow_ptr = ws.vrow_ptr; a.vmap = ws.vmap; a.part = ws.part; a.vcap = ws.vcap;
  const int grid = d->num_sms;
  const bool sin = d->cfg.sin_embedding != 0, det = d->deterministic != 0;
  switch (H) {
    case 64: run_gcl<64>(a, sin, det, grid, s); break;
    case 128: run_gcl<128>(a, sin, det, grid, s); break;
    case 192: run_gcl<192>(a, sin, det, grid, s); break;
    case 256: run_gcl<256>(a, sin, det, grid, s); break;
    default: return DSB_ERR_UNSUPPORTED_CONFIG;
  }
  DSB_CUDA_OK(cudaGetLastError());
  return 0;
}

int launch_edge_coord(const dsb_dynamics* d, const Dims& dm, const Workspace& ws, const EquivW& w,
                      const float4* x, PView pv, cudaStream_t s) {
  const dsb_config& c = d->cfg;
  const int H = c.hidden_nf;
  EdgeCoordArgs a;
  a.nm = c.reflection_equivariant ? 1 : 2;
  a.P = pv.P; a.ldp = pv.ldp; a.x = x; a.cent = ws.cent; a.gid = ws.gid;
  a.row_ptr = ws.row_ptr; a.n_rows = dm.n_coord_rows;
  a.erow = ws.erow; a.ecol = ws.ecol; a.ed0 = ws.ed0; a.NL = dm.NL; a.w = w;
  a.norm_constant = c.norm_constant; a.coords_range = c.coords_range; a.use_tanh = c.tanh;
  a.xagg = ws.xagg;
  a.vrow_ptr = ws.vrow_ptr; a.vmap = ws.vmap; a.part = reinterpret_cast<float4*>(ws.part); a.vcap = ws.vcap;
  const int grid = d->num_sms;
  const bool sin = c.sin_embedding != 0, det = d->deterministic != 0;
  switch (H) {
    case 64: run_coord<64>(a, sin, det, grid, s); break;
    case 128: run_coord<128>(a, sin, det, grid, s); break;
    case 192: run_coord<192>(a, sin, det, grid, s); break;
    case 256: run_coord<256>(a, sin, det, grid, s); break;
    default: return DSB_ERR_UNSUPPORTED_CONFIG;
  }
  DSB_CUDA_OK(cudaGetLastError());
  return 0;
}

// =====================================================================================================
// deterministic mode: fixed-order receiver sums from the chunk partials of the edge kernels.  One thread per (receiver,
// float4 column group); it adds the receiver's slots one after another in ascending order, so the result is a function of
// the slot contents alone (no atomics, no dependence on the grid).
__global__ void __launch_bounds__(256) segment_reduce_kernel(const float4* __restrict__ part, int ld4,
                                                             const int32_t* __restrict__ vrow_ptr, int vcap, int n_rows,
                                                             int spc, float4* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n_rows * ld4) return;
  const int i = (int)(idx / ld4), c = (int)(idx - (int64_t)i * ld4);
  const int k0 = (min(vrow_ptr[i], vcap) / kRowChunk) * spc, k1 = (min(vrow_ptr[i + 1], vcap) / kRowChunk) * spc;
  float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int k = k0; k < k1; ++k) {
    const float4 v = part[(size_t)k * ld4 + c];
    sum.x += v.x; sum.y += v.y; sum.z += v.z; sum.w += v.w;
  }
  out[(size_t)i * ld4 + c] = sum;
}

int launch_segment_reduce(const Workspace& ws, int n_rows, int ld4, int spc, float4* out, cudaStream_t s) {
  if (n_rows == 0) return 0;
  const int64_t tot = (int64_t)n_rows * ld4;
  DSB_CUDA_OK(launch_k(segment_reduce_kernel, (unsigned)((tot + 255) / 256), 256, 0, s,
                       reinterpret_cast<const float4*>(ws.part), ld4, (const int32_t*)ws.vrow_ptr, (int)ws.vcap, n_rows, spc, out));
  return 0;
}

}  // namespace dsb
