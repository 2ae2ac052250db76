// Tensor-core (wgmma, sm_90a) kernels of the denoiser: 3-product split contractions (3xFP16 or 3xTF32 operands), or the
// single fp16 product (1xFP16), with fp32 accumulation in registers.
//
//   tc_node_gemm_kernel    — C = act([A1 | A2/div] @ W + bias) (+R)   (node MLPs, merged first layers)
//   tc_edge_kernel<0,..>   — GCL.edge_model + receiver sums           (egnn_new.py:31-52)
//   tc_edge_kernel<1,..>   — EquivariantUpdate.coord_model            (egnn_new.py:96-116)
//
// One persistent CTA per SM with two MMA warpgroups and one weight warpgroup.  A 128-row tile is split between the MMA
// warpgroups (64 rows each = M of one wgmma, N = H).  Per K-chunk each builds its rows of the A operand (hi/lo split,
// 128B-swizzled) in shared memory, issues 4 k-steps x 3 split products asynchronously and builds the next chunk while they
// run.  The weight chunks (pre-split, pre-swizzled images) arrive by bulk copies into a two-stage ring, issued by one
// thread of the weight warpgroup.  The epilogue works on the accumulator registers directly (a thread holds rows r, r + 8
// and the column pairs 8j + 2 (lane % 4)).
#include "dsb_tc.cuh"

namespace dsb {
using namespace tc;

// =====================================================================================================
// weight images: B[n][k] (= the reference's own [out][in] Linear layout) split into hi/lo and laid out as
// [n_tile][k_chunk][H rows x 128 B, SWIZZLE_128B] (n-tiles are H = hidden_nf wide) so that one k-chunk is a single bulk copy.
// =====================================================================================================
__global__ void pack_b_image_kernel(float* __restrict__ hi, float* __restrict__ lo, const float* __restrict__ src, int lds,
                                    int scol, int n_rows, int n_dst_off, int K, int chunks, int TN) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n_rows * K) return;
  const int n = (int)(idx / K), k = (int)(idx - (int64_t)n * K);
  const int nd = n_dst_off + n, nt = nd / TN, nl = nd % TN;
  const int kc = k / TKC, c = (k % TKC) >> 2, j = k & 3;
  const size_t off = ((size_t)nt * chunks + kc) * (size_t)(TN * TKC) + sw128_offset(nl, c) / 4 + j;
  const float w = src[(size_t)n * lds + scol + k];
  const float h = tf32_hi(w);
  hi[off] = h;
  lo[off] = w - h;
}

void launch_pack_b_image(float* hi, float* lo, const float* src, int lds, int scol, int n_rows, int n_dst_off, int K, int tn) {
  const int64_t tot = (int64_t)n_rows * K;
  pack_b_image_kernel<<<(unsigned)((tot + 255) / 256), 256>>>(hi, lo, src, lds, scol, n_rows, n_dst_off, K, K / TKC, tn);
}

// 3xFP16 images: w*scale = w_h + w_l in fp16, [n_tile][K/64][256 rows x 128 B (64 halfs), SWIZZLE_128B]
__global__ void pack_b_image_f16_kernel(__half* __restrict__ hi, __half* __restrict__ lo, const float* __restrict__ src, int lds,
                                        int scol, int n_rows, int n_dst_off, int K, int chunks, float scale, int TN) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n_rows * K) return;
  const int n = (int)(idx / K), k = (int)(idx - (int64_t)n * K);
  const int nd = n_dst_off + n, nt = nd / TN, nl = nd % TN;
  const int kc = k / TKC16, c16 = (k % TKC16) >> 3, j = k & 7;
  const size_t off = ((size_t)nt * chunks + kc) * (size_t)(TN * 64) + sw128_offset(nl, c16) / 2 + j;
  const float w = src[(size_t)n * lds + scol + k] * scale;
  const __half h = __float2half_rn(w);
  hi[off] = h;
  lo[off] = __float2half_rn(w - __half2float(h));
}

void launch_pack_b_image_f16(float* hi, float* lo, const float* src, int lds, int scol, int n_rows, int n_dst_off, int K, float scale, int tn) {
  const int64_t tot = (int64_t)n_rows * K;
  pack_b_image_f16_kernel<<<(unsigned)((tot + 255) / 256), 256>>>(reinterpret_cast<__half*>(hi), reinterpret_cast<__half*>(lo), src,
                                                                  lds, scol, n_rows, n_dst_off, K, K / TKC16, scale, tn);
}

// max |src[n][scol + k]| over an [n_rows][K] block -> *out (device uint holding the float bits; non-negative floats order as uints)
__global__ void absmax_kernel(const float* __restrict__ src, int lds, int scol, int n_rows, int K, unsigned* __restrict__ out) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  float v = 0.f;
  if (idx < (int64_t)n_rows * K) { const int n = (int)(idx / K), k = (int)(idx - (int64_t)n * K); v = fabsf(src[(size_t)n * lds + scol + k]); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(v));
}
void launch_absmax(const float* src, int lds, int scol, int n_rows, int K, unsigned* out) {
  const int64_t tot = (int64_t)n_rows * K;
  absmax_kernel<<<(unsigned)((tot + 255) / 256), 256>>>(src, lds, scol, n_rows, K, out);
}

// ---- common prologue -------------------------------------------------------------------------------------------------
constexpr size_t kControlBytes = 128;      // keeps the per-kernel extras 16-byte aligned for float4 access
static_assert(sizeof(Control) <= kControlBytes, "Control block grew");
__device__ __forceinline__ char* align1024(uint8_t* raw) {
  return reinterpret_cast<char*>(raw) + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
}
template <int H> constexpr size_t tc_smem_base() { return 1024 + (size_t)NSTAGE * Geo<H>::STAGE_BYTES + kControlBytes; }

// =====================================================================================================
// node GEMM: C = act([A1 | A2/div] @ W + bias) (+R), one 128 x H output tile per work item
// =====================================================================================================
struct TcGemmArgs {
  const float* A1; int lda1; int K1;
  const float* A2; int lda2; int K2; float div2; const int32_t* deg2;     // deg2 != nullptr: per-row divisor max(deg2[m], 1) ('mean')
  const float* Bhi; const float* Blo;        // [Nn/H][K/kc][H rows x 128 B] images
  const float* bias; const float* R; int ldr;
  float* C; int ldc; int M; int Nn; int act;
  float* Z; int ldz;
  int dead_mt; int dead_nt;                    // tiles with m-tile >= dead_mt and n-tile < dead_nt are skipped (dead_nt == 0: none)
  float inv_scale;                             // 3xFP16 / 1xFP16: 1 / (X_SCALE * weight scale); 1 for 3xTF32
};

// live-tile enumeration: region A = m-tiles [0, dead_mt) x all n-tiles, region B = m-tiles [dead_mt, ntm) x n-tiles [dead_nt, ntn)
struct TileMap {
  int ntn, ntm, dead_mt, dead_nt, nA, n_live;
  __device__ TileMap(int M, int Nn, int dmt, int dnt, int TN) {
    ntn = Nn / TN; ntm = (M + TM - 1) / TM;
    dead_nt = dnt; dead_mt = dnt > 0 ? (dmt < ntm ? dmt : ntm) : ntm;
    nA = dead_mt * ntn;
    n_live = nA + (ntm - dead_mt) * (ntn - dead_nt);
  }
  __device__ void get(int t, int& mt, int& nt) const {
    if (t < nA) { mt = t / ntn; nt = t - mt * ntn; }
    else { const int u = t - nA, w = ntn - dead_nt; mt = dead_mt + u / w; nt = dead_nt + (u - (u / w) * w); }
  }
};

template <TcFormat FMT, int H>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_node_gemm_kernel(TcGemmArgs g) {
  using G = Geo<H>;
  constexpr bool F16 = FMT != TcFormat::TF32x3;
  constexpr int TN = H, HPC = F16 ? 2 : 1;     // 32-k halves per pipeline chunk
  extern __shared__ uint8_t smem_raw[];
  char* const stages = align1024(smem_raw);
  Control* ctl = reinterpret_cast<Control*>(stages + NSTAGE * G::STAGE_BYTES);
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const TileMap tm(g.M, g.Nn, g.dead_mt, g.dead_nt, TN);
  const int n_tiles = tm.n_live;
  const int n_my = ((int)blockIdx.x < n_tiles) ? (n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
  if (n_my == 0) return;
  const int K = g.K1 + g.K2, chunks = K / (F16 ? TKC16 : TKC);
  const uint32_t total = (uint32_t)(n_my * chunks);
  pdl_trigger();
  if (threadIdx.x == 0) control_init(ctl);
  __syncthreads();
  pdl_wait();
  const WeightStream<FMT, H> wst{ctl, stages};
  auto issue_w = [&](uint32_t q) {             // weight chunk of global chunk index q
    const int it = (int)(q / chunks), kc = (int)(q - (uint32_t)it * chunks);
    int mt, nt;
    tm.get(blockIdx.x + it * gridDim.x, mt, nt);
    const size_t off = ((size_t)nt * chunks + kc) * G::B_CHUNK_FLOATS;
    wst.issue(q, g.Bhi + off, g.Blo + off);
  };
  if (threadIdx.x >= MMA_THREADS) {            // weight warpgroup: the whole chunk sequence, two stages ahead at most
    regs_dec<WEIGHT_WG_REGS>();
    if (threadIdx.x == MMA_THREADS)
      for (uint32_t q = 0; q < total; ++q) issue_w(q);
    return;
  }
  regs_inc<MMA_WG_REGS>();

  // producer mapping (coalesced loads): warp owns 16 rows of its warpgroup's 64; lane = (sub-row sr, 16-byte piece pc)
  const int sr = lane >> 3, pc = lane & 7;
  const int r0 = wg * WG_ROWS + 16 * warp + 4 * sr;        // first of this thread's four tile rows
  const int re = wg * WG_ROWS + 16 * warp + (lane >> 2);   // accumulator rows re, re + 8
  const bool divides = g.div2 != 1.0f || g.deg2 != nullptr;
  float acc[G::ACC];
  MmaTracker trk;
  uint32_t q = 0;
  for (int it = 0; it < n_my; ++it) {
    int mt, nt;
    tm.get(blockIdx.x + it * gridDim.x, mt, nt);
    const int m0 = mt * TM, n0 = nt * TN;
    for (int kc = 0; kc < chunks; ++kc, ++q) {
      const int s = q & 1;
      char* st = stages + (size_t)s * G::STAGE_BYTES;
#pragma unroll
      for (int h = 0; h < HPC; ++h) {
        const int hf = kc * HPC + h, k = hf * TKC + 4 * pc;
        const bool second = k >= g.K1;
        float4 v[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int m = m0 + r0 + i;
          v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (m < g.M) v[i] = second ? *reinterpret_cast<const float4*>(g.A2 + (size_t)m * g.lda2 + (k - g.K1))
                                     : *reinterpret_cast<const float4*>(g.A1 + (size_t)m * g.lda1 + k);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float4 x = v[i];
          if (second && divides) {             // columns of A2: exact division by the normalisation
            const int m = m0 + r0 + i;
            const float dv = g.deg2 ? (float)max(m < g.M ? g.deg2[m] : 1, 1) : g.div2;
            x.x = __fdiv_rn(x.x, dv); x.y = __fdiv_rn(x.y, dv); x.z = __fdiv_rn(x.z, dv); x.w = __fdiv_rn(x.w, dv);
          }
          store_pair<FMT>(st + piece_offset<F16>(r0 + i, hf, pc), pk2(x.x, x.y), pk2(x.z, x.w));
        }
      }
      fence_proxy_async();                     // generic-proxy operand stores -> visible to the wgmma (async proxy)
      wg_sync(wg);
      mbar_wait(&ctl->full_w[s], (q >> 1) & 1);
      wgmma_fence();
      mma_chunk<FMT, H>(acc, st, wg, kc == 0);
      wgmma_commit();
      trk.release_prev(ctl, (int)q, lane == 0);
    }
    trk.drain<H>(ctl, acc, lane == 0);
    // epilogue from registers: rows re, re + 8; columns 8j + 2 (lane % 4) + {0, 1}
    const f32x2 ip = pk2(g.inv_scale, g.inv_scale);
#pragma unroll
    for (int j = 0; j < H / 8; ++j) {
      const int n = n0 + 8 * j + 2 * (lane & 3);
      const f32x2 b = g.bias ? *reinterpret_cast<const float2*>(g.bias + n) : pk2(0.f, 0.f);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        f32x2 x = pk2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);      // read outside the row test: the accumulators
        x = F16 ? fma2(x, ip, b) : add2(x, b);                             // are not used on a divergent path
        if (g.act == 1) x = silu2(x);
        upk2(x, acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);
      }
    }
    // Residual: every R load is issued before the first store.  R and C may be the same buffer (g3: h += ...), so the
    // compiler keeps loads and stores in program order; read inside the store loop, each load would wait for the
    // previous store and the epilogue would pay H / 4 dependent L2 round trips.  Rows past M read row M - 1 (no branch
    // next to the accumulators) and are not stored.
    if (g.R) {
#pragma unroll
      for (int j = 0; j < H / 8; ++j) {
        const int n = n0 + 8 * j + 2 * (lane & 3);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = min(m0 + re + 8 * hh, g.M - 1);
          const f32x2 x = add2(*reinterpret_cast<const float2*>(g.R + (size_t)row * g.ldr + n),
                               pk2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]));
          upk2(x, acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);
        }
      }
    }
    acc_fence(acc);
#pragma unroll
    for (int j = 0; j < H / 8; ++j) {
      const int n = n0 + 8 * j + 2 * (lane & 3);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int row = m0 + re + 8 * hh;
        if (row < g.M) {
          *reinterpret_cast<float2*>(g.C + (size_t)row * g.ldc + n) = pk2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);
          if (g.Z) *reinterpret_cast<float2*>(g.Z + (size_t)row * g.ldz + n) = make_float2(0.f, 0.f);
        }
      }
    }
  }
}

// =====================================================================================================
// edge kernels
// =====================================================================================================
struct EdgeScalars {          // per-edge scalars of one unit (virtual row order)
  float d2[TM], d0[TM];
  int row[TM], col[TM], type[TM];
  float dir[3][TM];           // coord: direction of this MLP's term
};

template <int H>
struct EdgeExtra {            // shared memory after Control
  float vec[2][3 * H];        // per MLP: wr, wr0, b2   (the edge-type table tb stays in global/L1)
  float wa[H];                // attention weight (GCL) or w3 (coord)
  EdgeScalars sc[2];          // unit j uses sc[j & 1]; unit j + 1's are written while unit j is on the tensor pipe
};

struct TcEdgeArgs {
  const float* P; int ldp;
  const float4* x; const float4* cent; const int32_t* gid;
  const int32_t* vrow_ptr; const int32_t* vmap; int n_rows;   // virtual rows [0, vrow_ptr[n_rows]): vmap[v] = edge index or -1 (pad)
  const int32_t *erow, *ecol; const float* ed0; int NL;
  int nm;                                    // MLPs per edge tile: 1 (GCL, reflection-equivariant coord) or 2 (coord + cross)
  const float* W2hi[2]; const float* W2lo[2];   // [H/kc][H rows x 128 B] images
  const float* wr[2]; const float* wr0[2]; const float* tb[2]; const float* b2[2];
  const float* wa; const float* ba;          // GCL attention (nullptr: none) / coord: wa = w3
  float norm_constant, coords_range; int use_tanh;
  float* agg;                                // GCL: [N][H] raw sums
  float4* xagg;                              // coord: [N] raw sums of trans
  float inv_scale[2];                        // 3xFP16 / 1xFP16: 1 / (X_SCALE * W2 scale) per MLP; 1 for 3xTF32
  float* part;                               // deterministic variant: chunk partials (Workspace::part) instead of agg / xagg
  int vcap;                                  // deterministic variant: virtual rows covered by vmap / part (Workspace::vcap)
};

// Per-edge scalars of the unit at virtual row v0 for MLP m (thread pr handles virtual row v0 + pr), produced in four steps
// that each wait for the loads of the one before: 0 vmap, 1 edge ids and d0, 2 coordinates (and graph id), 3 centroid,
// finish and store.  The edge kernel runs the steps of the next unit between the chunks of the current one, so each load's
// latency hides under a chunk of wgmmas.  Branch-free (clamped indices, selects): it runs inside the wgmma window.
// Rows past V and pad rows (vmap -1) get row -1 and zero scalars.
template <bool COORD>
struct ScalarSteps {
  int e, r, c, gi;
  float d0;
  float4 xi, xj;
  __device__ __forceinline__ void step(int k, const TcEdgeArgs& a, EdgeScalars* sc, int pr, int v0, int V, int m) {
    if (k == 0) {
      const int vr = v0 + pr;
      e = a.vmap[min(vr, V - 1)];
      e = vr < V ? e : -1;
    } else if (k == 1) {
      const int ec = max(e, 0);
      r = a.erow[ec]; c = a.ecol[ec]; d0 = a.ed0[ec];
      r = e >= 0 ? r : 0; c = e >= 0 ? c : 0;
    } else if (k == 2) {
      xi = a.x[r]; xj = a.x[c];
      if (COORD) gi = a.gid[r];
    } else {
      const bool live = e >= 0;
      const float dx = xi.x - xj.x, dy = xi.y - xj.y, dz = xi.z - xj.z;
      const float d2 = dx * dx + dy * dy + dz * dz;
      const int ty = (r < a.NL) == (c < a.NL) ? (r < a.NL ? 1 : 2) : 0;
      sc->row[pr] = live ? r : -1; sc->col[pr] = c; sc->d2[pr] = live ? d2 : 0.f; sc->d0[pr] = live ? d0 : 0.f;
      sc->type[pr] = live ? ty : 0;
      if (COORD) {
        float dir[3];
        if (m == 0) {                                                   // egnn_new.py:300-301 (coord2diff)
          const float den = sqrtf(d2 + 1e-8f) + a.norm_constant;
          dir[0] = dx / den; dir[1] = dy / den; dir[2] = dz / den;
        } else {                                                        // egnn_new.py:312-315 (coord2cross)
          const float4 mu = a.cent[gi];
          const float ax = xi.x - mu.x, ay = xi.y - mu.y, az = xi.z - mu.z;
          const float bx = xj.x - mu.x, by = xj.y - mu.y, bz = xj.z - mu.z;
          const float cx = ay * bz - az * by, cy = az * bx - ax * bz, cz = ax * by - ay * bx;
          const float cn = sqrtf(cx * cx + cy * cy + cz * cz) + a.norm_constant;
          dir[0] = cx / cn; dir[1] = cy / cn; dir[2] = cz / cn;
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) sc->dir[k][pr] = live ? dir[k] : 0.f;
      }
    }
  }
};

// Work unit = virtual tile v = edge_tile * nm + m (the m-th MLP over 128 virtual edge rows).  The coordinate update is a sum
// of independent terms per MLP (egnn_new.py:100-109: trans = diff * f(phi) + cross * f(phi_x)), so the two MLPs of an edge tile
// are independent units that add into the same receiver sums; units are dealt round-robin to the CTAs.
//
// Per unit and warpgroup (64 virtual edge rows): per-edge scalars -> for each K-chunk: A operand = SiLU(P[recv] + P[send] +
// d^2 wr + d0^2 wr0 (+ tb[type])) split into hi/lo and stored swizzled, wgmmas against the streamed W2 chunk -> epilogue:
// m = SiLU(acc + b2), s = wa . m per row (four lanes share a row: two shuffles), then
//   GCL:   agg[recv] += gate * m, gate = sigmoid(s + ba) (1 without attention); receiver segments start at multiples of
//          kRowChunk = 4 virtual rows, so the 4 rows of a chunk (lanes 4 and 8 apart) are summed by shuffles and one lane
//          per chunk and column pair issues a vector RED;
//   coord: xagg[recv] += dir * f(s) (egnn_new.py:100-109), chunk sums by shuffles, one atomic per chunk and component.
// DET (deterministic mode): the same chunk sums are stored, not added, into slot (virtual chunk) of a.part (coord: slot
// chunk * nm + m, one float4); launch_segment_reduce then sums each receiver's slots in ascending order.  The chunk sums
// have a fixed content and order, so the receiver sums depend on the receiver's own edges only.
template <bool COORD, TcFormat FMT, int H, bool TB, bool DET = false>
__global__ void __launch_bounds__(TC_THREADS, 1) tc_edge_kernel(TcEdgeArgs a) {
  using G = Geo<H>;
  constexpr bool F16 = FMT != TcFormat::TF32x3;
  constexpr int HPC = F16 ? 2 : 1;             // 32-k halves per pipeline chunk
  constexpr int chunks = H / (TKC * HPC);
  extern __shared__ uint8_t smem_raw[];
  char* const stages = align1024(smem_raw);
  Control* ctl = reinterpret_cast<Control*>(stages + NSTAGE * G::STAGE_BYTES);
  EdgeExtra<H>* ex = reinterpret_cast<EdgeExtra<H>*>(reinterpret_cast<char*>(ctl) + kControlBytes);
  const int wg = threadIdx.x >> 7, wt = threadIdx.x & 127, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int nm = a.nm;

  pdl_trigger();
  for (int i = threadIdx.x; i < H; i += TC_THREADS) {
    for (int m = 0; m < nm; ++m) {
      float* v = ex->vec[m];
      v[i] = a.wr[m][i]; v[H + i] = a.wr0[m][i]; v[2 * H + i] = a.b2[m][i];
    }
    ex->wa[i] = a.wa ? a.wa[i] : 0.f;
  }
  if (threadIdx.x == 0) control_init(ctl);
  __syncthreads();
  pdl_wait();                 // everything above touches only kernel arguments and constant weights
  // virtual rows: every receiver's edges start at a multiple of kRowChunk (DET: never past the partial buffer)
  const int E = DET ? min(a.vrow_ptr[a.n_rows], a.vcap) : a.vrow_ptr[a.n_rows];
  const int n_units = ((E + TM - 1) / TM) * nm;
  const int n_my = ((int)blockIdx.x < n_units) ? (n_units - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
  if (n_my == 0) return;
  auto unit_tile = [&](int j, int& m) { const int v = blockIdx.x + j * gridDim.x, t = v / nm; m = v - t * nm; return t; };
  const uint32_t total = (uint32_t)(n_my * chunks);
  const WeightStream<FMT, H> wst{ctl, stages};
  auto issue_w = [&](uint32_t q) {
    const int j = (int)(q / chunks), kc = (int)(q - (uint32_t)j * chunks);
    int m;
    unit_tile(j, m);
    wst.issue(q, a.W2hi[m] + (size_t)kc * G::B_CHUNK_FLOATS, a.W2lo[m] + (size_t)kc * G::B_CHUNK_FLOATS);
  };
  if (threadIdx.x >= MMA_THREADS) {            // weight warpgroup: the whole chunk sequence, two stages ahead at most
    regs_dec<WEIGHT_WG_REGS>();
    if (threadIdx.x == MMA_THREADS)
      for (uint32_t q = 0; q < total; ++q) issue_w(q);
    return;
  }
  regs_inc<MMA_WG_REGS>();

  const bool has_att = (!COORD) && a.wa != nullptr;
  const float ba = has_att ? a.ba[0] : 0.f;
  // producer mapping: warp owns 16 rows of its warpgroup's 64; lane = (sub-row sr, 16-byte piece pc).  A thread handles the
  // 4-row chunk r0 .. r0 + 3, which belongs to one receiver: the receiver operand P[recv] is one load per half.
  const int sr = lane >> 3, pc = lane & 7;
  const int r0 = wg * WG_ROWS + 16 * warp + 4 * sr;
  const int re = wg * WG_ROWS + 16 * warp + (lane >> 2);   // accumulator rows re, re + 8
  const float* const Pt = a.P + 4 * pc;
  const int soff = nm * H;                   // sender block follows the nm receiver blocks
  // A operand of K-chunk kc of the unit with scalars sc and MLP m into stage s
  auto build = [&](const EdgeScalars* sc, int m, int kc, int s) {
    char* st = stages + (size_t)s * G::STAGE_BYTES;
    const int moff = m * H;
    const float* pr = Pt + (size_t)max(sc->row[r0], 0) * a.ldp + moff;
    const int4 cl = *reinterpret_cast<const int4*>(sc->col + r0);
    const float4 d2v = *reinterpret_cast<const float4*>(sc->d2 + r0), d0v = *reinterpret_cast<const float4*>(sc->d0 + r0);
    const int4 tyv = *reinterpret_cast<const int4*>(sc->type + r0);
    const float* const ps[4] = {Pt + (size_t)cl.x * a.ldp + (soff + moff), Pt + (size_t)cl.y * a.ldp + (soff + moff),
                                Pt + (size_t)cl.z * a.ldp + (soff + moff), Pt + (size_t)cl.w * a.ldp + (soff + moff)};
    const float pd2[4] = {d2v.x, d2v.y, d2v.z, d2v.w}, pd0[4] = {d0v.x, d0v.y, d0v.z, d0v.w};
    const int pty[4] = {TB ? tyv.x * H : 0, TB ? tyv.y * H : 0, TB ? tyv.z * H : 0, TB ? tyv.w * H : 0};
    const float* wr = ex->vec[m] + 4 * pc;
    const float* wr0 = wr + H;
    const float* tbm = TB ? a.tb[m] + 4 * pc : nullptr;
#pragma unroll
    for (int h = 0; h < HPC; ++h) {
      const int hf = kc * HPC + h;
      const float4 ga = *reinterpret_cast<const float4*>(pr + hf * TKC);
      float4 gb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) gb[i] = *reinterpret_cast<const float4*>(ps[i] + hf * TKC);
      const float4 r4 = *reinterpret_cast<const float4*>(wr + hf * TKC);
      const float4 r04 = *reinterpret_cast<const float4*>(wr0 + hf * TKC);
      const f32x2 a01 = pk2(ga.x, ga.y), a23 = pk2(ga.z, ga.w);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const f32x2 d2p = pk2(pd2[i], pd2[i]), d0p = pk2(pd0[i], pd0[i]);
        f32x2 u01 = fma2(d0p, pk2(r04.x, r04.y), fma2(d2p, pk2(r4.x, r4.y), add2(a01, pk2(gb[i].x, gb[i].y))));
        f32x2 u23 = fma2(d0p, pk2(r04.z, r04.w), fma2(d2p, pk2(r4.z, r4.w), add2(a23, pk2(gb[i].z, gb[i].w))));
        if (TB) {
          const float4 t4 = *reinterpret_cast<const float4*>(tbm + pty[i] + hf * TKC);
          u01 = add2(u01, pk2(t4.x, t4.y)); u23 = add2(u23, pk2(t4.z, t4.w));
        }
        silu_pair<(DSB_SILU_PAIR & 1) != 0, (DSB_SILU_QUAD & 1) != 0>(u01, u23);
        store_pair<FMT>(st + piece_offset<F16>(r0 + i, hf, pc), u01, u23);
      }
    }
  };
  float acc[G::ACC];
  MmaTracker trk;
  uint32_t q = 0;
  // issue the wgmmas of chunk kc (global chunk q, built into stage q & 1)
  auto issue = [&](int kc) {
    const int s = q & 1;
    fence_proxy_async();
    wg_sync(wg);
    mbar_wait(&ctl->full_w[s], (q >> 1) & 1);
    wgmma_fence();
    mma_chunk<FMT, H>(acc, stages + (size_t)s * G::STAGE_BYTES, wg, kc == 0);
    wgmma_commit();
    trk.release_prev(ctl, (int)q, lane == 0);
    ++q;
  };
  // Unit pipeline: unit j + 1's scalars are produced into sc[(j + 1) & 1] step by step after chunks 0 .. chunks - 2 of unit
  // j have been issued, and its chunk 0 is built under unit j's last chunk; only the epilogue runs with no wgmma in flight.
  // Both threads of a row pair (wt, wt + 64) produce the row's scalars (same values): no thread-dependent branch.
  static_assert(chunks >= 2, "the scalar steps of the next unit need at least one chunk before the last");
  constexpr int kSteps = 4;
  const int psc = wg * WG_ROWS + (wt & (WG_ROWS - 1));
  ScalarSteps<COORD> stp;
  int m;
  int e0 = unit_tile(0, m) * TM;
  for (int k = 0; k < kSteps; ++k) stp.step(k, a, &ex->sc[0], psc, e0, E, m);
  wg_sync(wg);
  build(&ex->sc[0], m, 0, 0);
  for (int j = 0; j < n_my; ++j) {
    const EdgeScalars* sc = &ex->sc[j & 1];
    EdgeScalars* sc_next = &ex->sc[(j + 1) & 1];
    int m_next;
    const int e0_next = unit_tile(j + 1, m_next) * TM;      // past the last unit: rows >= E, all padding
    // the 1xFP16 GCL kernel at H = 256 with the type table stays rolled: fully unrolled, ptxas spills there
#pragma unroll ((F16 && !(FMT == TcFormat::F16x1 && !COORD && TB && H == 256)) ? chunks : 1)
    for (int kc = 0; kc < chunks - 1; ++kc) {
      issue(kc);
      for (int k = kc * kSteps / (chunks - 1); k < (kc + 1) * kSteps / (chunks - 1); ++k)
        stp.step(k, a, sc_next, psc, e0_next, E, m_next);
      build(sc, m, kc + 1, q & 1);
    }
    issue(chunks - 1);
    build(sc_next, m_next, 0, q & 1);
    trk.drain<H>(ctl, acc, lane == 0);

    // ---- epilogue, pass 1: m = SiLU(acc * inv + b2) in place; s = wa . m per row
    const float* b2 = ex->vec[m] + 2 * H;
    const f32x2 ip = pk2(a.inv_scale[m], a.inv_scale[m]);
    float s_lo = 0.f, s_hi = 0.f;
    if constexpr (DET) {
      // Batch-invariant grouping: the shared-reciprocal SiLU takes column groups jj and jj + 1 of ONE row (re, then re + 8),
      // so an edge's messages depend on that edge alone, not on the edge 8 rows away (which changes with the batch layout).
      // Same number of SiLU calls as below; the row sums s keep their column order.
      static_assert((H / 8) % 2 == 0, "DET epilogue pairs column groups");
#pragma unroll
      for (int jj = 0; jj < H / 8; jj += 2) {
        const int c = 8 * jj + 2 * (lane & 3);
        const f32x2 b0 = *reinterpret_cast<const float2*>(b2 + c), b1 = *reinterpret_cast<const float2*>(b2 + c + 8);
        const float2 w0 = *reinterpret_cast<const float2*>(ex->wa + c), w1 = *reinterpret_cast<const float2*>(ex->wa + c + 8);
        f32x2 lo0 = pk2(acc[4 * jj], acc[4 * jj + 1]), lo1 = pk2(acc[4 * jj + 4], acc[4 * jj + 5]);
        f32x2 hi0 = pk2(acc[4 * jj + 2], acc[4 * jj + 3]), hi1 = pk2(acc[4 * jj + 6], acc[4 * jj + 7]);
        lo0 = F16 ? fma2(lo0, ip, b0) : add2(lo0, b0); lo1 = F16 ? fma2(lo1, ip, b1) : add2(lo1, b1);
        hi0 = F16 ? fma2(hi0, ip, b0) : add2(hi0, b0); hi1 = F16 ? fma2(hi1, ip, b1) : add2(hi1, b1);
        silu_pair<(DSB_SILU_PAIR & 2) != 0, (DSB_SILU_QUAD & 2) != 0>(lo0, lo1);
        silu_pair<(DSB_SILU_PAIR & 2) != 0, (DSB_SILU_QUAD & 2) != 0>(hi0, hi1);
        upk2(lo0, acc[4 * jj], acc[4 * jj + 1]); upk2(lo1, acc[4 * jj + 4], acc[4 * jj + 5]);
        upk2(hi0, acc[4 * jj + 2], acc[4 * jj + 3]); upk2(hi1, acc[4 * jj + 6], acc[4 * jj + 7]);
        s_lo = fmaf(lo0.y, w0.y, fmaf(lo0.x, w0.x, s_lo));
        s_lo = fmaf(lo1.y, w1.y, fmaf(lo1.x, w1.x, s_lo));
        s_hi = fmaf(hi0.y, w0.y, fmaf(hi0.x, w0.x, s_hi));
        s_hi = fmaf(hi1.y, w1.y, fmaf(hi1.x, w1.x, s_hi));
      }
    } else {
#pragma unroll
    for (int jj = 0; jj < H / 8; ++jj) {
      const int c = 8 * jj + 2 * (lane & 3);
      const f32x2 bb = *reinterpret_cast<const float2*>(b2 + c);
      const float2 ww = *reinterpret_cast<const float2*>(ex->wa + c);
      f32x2 lo = pk2(acc[4 * jj], acc[4 * jj + 1]), hi = pk2(acc[4 * jj + 2], acc[4 * jj + 3]);
      lo = F16 ? fma2(lo, ip, bb) : add2(lo, bb);
      hi = F16 ? fma2(hi, ip, bb) : add2(hi, bb);
      silu_pair<(DSB_SILU_PAIR & 2) != 0, (DSB_SILU_QUAD & 2) != 0>(lo, hi);
      upk2(lo, acc[4 * jj], acc[4 * jj + 1]); upk2(hi, acc[4 * jj + 2], acc[4 * jj + 3]);
      s_lo = fmaf(lo.y, ww.y, fmaf(lo.x, ww.x, s_lo));
      s_hi = fmaf(hi.y, ww.y, fmaf(hi.x, ww.x, s_hi));
    }
    }
    s_lo += __shfl_xor_sync(0xffffffffu, s_lo, 1); s_lo += __shfl_xor_sync(0xffffffffu, s_lo, 2);
    s_hi += __shfl_xor_sync(0xffffffffu, s_hi, 1); s_hi += __shfl_xor_sync(0xffffffffu, s_hi, 2);
    const int row_lo = sc->row[re], row_hi = sc->row[re + 8];
    const int crow_lo = sc->row[re & ~3], crow_hi = sc->row[(re + 8) & ~3];     // receiver of the row's 4-row chunk
    const bool chunk_lane = (lane & 12) == 0;                                   // first row of its chunk
    if constexpr (!COORD) {
      // ---- pass 2: gate-weighted messages, 4-row chunk sums (reduce-scatter), one vector RED per lane and column-group pair
      // pad rows share a chunk with real rows: weight 0 (selects, not branches: a divergent path next to the accumulator
      // registers makes the compiler serialise the wgmmas)
      float g_lo = has_att ? sigmoid_f(s_lo + ba) : 1.0f, g_hi = has_att ? sigmoid_f(s_hi + ba) : 1.0f;
      g_lo = row_lo >= 0 ? g_lo : 0.f;
      g_hi = row_hi >= 0 ? g_hi : 0.f;
      // The four lanes of a chunk (lanes 4 and 8 apart) hold rows re (chunk lo) and re + 8 (chunk hi) of two column groups
      // jj, jj + 1: 8 values each.  Lanes 4 apart (rows 0|1, 2|3 of the chunks) swap halves and add: the lane with
      // (lane & 4) == 0 keeps chunk lo, its partner chunk hi.  Lanes 8 apart (row pairs {0,1}|{2,3}) swap again: the lane
      // with (lane & 8) == 0 keeps group jj, its partner group jj + 1.  Every lane ends with one finished column pair, summed
      // (x0 + x1) + (x2 + x3) over the chunk's rows as by the all-reduce this replaces.
      const bool hi_half = (lane & 4) != 0, odd_group = (lane & 8) != 0;
      const int crow = hi_half ? crow_hi : crow_lo;
      const int chunk_row = hi_half ? (re + 8) & ~3 : re & ~3;
      float* const dst = (DET ? a.part + (size_t)((e0 + chunk_row) / kRowChunk) * H : a.agg + (size_t)max(crow, 0) * H)
                         + 2 * (lane & 3) + (odd_group ? 8 : 0);
#pragma unroll
      for (int jj = 0; jj < H / 8; jj += 2) {
        const float lo[4] = {g_lo * acc[4 * jj], g_lo * acc[4 * jj + 1], g_lo * acc[4 * jj + 4], g_lo * acc[4 * jj + 5]};
        const float hi[4] = {g_hi * acc[4 * jj + 2], g_hi * acc[4 * jj + 3], g_hi * acc[4 * jj + 6], g_hi * acc[4 * jj + 7]};
        float t[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) t[k] = (hi_half ? hi[k] : lo[k]) + __shfl_xor_sync(0xffffffffu, hi_half ? lo[k] : hi[k], 4);
        float u[2];
#pragma unroll
        for (int k = 0; k < 2; ++k) u[k] = (odd_group ? t[2 + k] : t[k]) + __shfl_xor_sync(0xffffffffu, odd_group ? t[k] : t[2 + k], 8);
        // a chunk of padding only has gate 0 on all rows: its sums are exactly 0 and go to row 0 (DET: to the pad chunk's
        // own slot, which no receiver reads)
        if constexpr (DET)
          asm volatile("st.global.v2.f32 [%0], {%1, %2};" ::"l"(dst + 8 * jj), "f"(u[0]), "f"(u[1]) : "memory");
        else
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst + 8 * jj), "f"(u[0]), "f"(u[1]) : "memory");
      }
    } else {
      // ---- coord: this unit's term of trans for rows re, re + 8 (egnn_new.py:100-109), chunk sums
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = re + 8 * hh;
        const float sv = hh ? s_hi : s_lo;
        const bool live = (hh ? row_hi : row_lo) >= 0;
        float tr[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const float d = sc->dir[k][r];
          float t;
          if (m == 0) t = a.use_tanh ? (d * tanhf(sv)) * a.coords_range : d * sv;       // coord_diff * tanh(phi) * range
          else t = d * (a.use_tanh ? tanhf(sv) * a.coords_range : sv);                     // coord_cross * (tanh(phi_x) * range)
          t = live ? t : 0.f;
          t += __shfl_xor_sync(0xffffffffu, t, 4);
          t += __shfl_xor_sync(0xffffffffu, t, 8);
          tr[k] = t;
        }
        const int crow = hh ? crow_hi : crow_lo;
        if constexpr (DET) {
          if (chunk_lane && (lane & 3) == 0)
            reinterpret_cast<float4*>(a.part)[(size_t)((e0 + (r & ~3)) / kRowChunk) * nm + m] = make_float4(tr[0], tr[1], tr[2], 0.f);
        } else if (chunk_lane && (lane & 3) == 0 && crow >= 0) {
#pragma unroll
          for (int k = 0; k < 3; ++k) atomicAdd(reinterpret_cast<float*>(a.xagg) + (size_t)crow * 4 + k, tr[k]);
        }
      }
    }
    m = m_next; e0 = e0_next;
  }
}

// =====================================================================================================
// launchers
// =====================================================================================================
template <int H> static size_t gemm_smem_bytes() { return tc_smem_base<H>(); }
template <int H> static size_t edge_smem_bytes() {
  static_assert(tc_smem_base<H>() + sizeof(EdgeExtra<H>) <= 232448, "edge kernel exceeds the 227 KB of shared memory per CTA");
  return tc_smem_base<H>() + sizeof(EdgeExtra<H>);
}

bool tc_width_supported(int H) { return H == 128 || H == 192 || H == 256; }

// run `fn.template operator()<H>()` for the run-time width
template <typename Fn>
static int dispatch_width(int H, Fn&& fn) {
  switch (H) {
    case 128: return fn.template operator()<128>();
    case 192: return fn.template operator()<192>();
    case 256: return fn.template operator()<256>();
    default: set_error("tensor-core kernels exist for hidden_nf 128, 192, 256 (got %d)", H); return DSB_ERR_UNSUPPORTED_CONFIG;
  }
}

// run `fn.template operator()<F, H>()` for the run-time operand format and width
template <typename Fn>
static int dispatch_tc(TcFormat f, int H, Fn&& fn) {
  return dispatch_width(H, [&]<int W>() -> int {
    switch (f) {
      case TcFormat::TF32x3: return fn.template operator()<TcFormat::TF32x3, W>();
      case TcFormat::F16x3: return fn.template operator()<TcFormat::F16x3, W>();
      default: return fn.template operator()<TcFormat::F16x1, W>();
    }
  });
}

int configure_tc_kernels(int H) {
  for (const TcFormat f : {TcFormat::TF32x3, TcFormat::F16x3, TcFormat::F16x1}) {
    const int e = dispatch_tc(f, H, [&]<TcFormat F, int W>() -> int {
      const int gs = (int)gemm_smem_bytes<W>(), es = (int)edge_smem_bytes<W>();
      DSB_CUDA_OK(cudaFuncSetAttribute(tc_node_gemm_kernel<F, W>, cudaFuncAttributeMaxDynamicSharedMemorySize, gs));
      DSB_CUDA_OK(cudaFuncSetAttribute(tc_edge_kernel<false, F, W, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, es));
      DSB_CUDA_OK(cudaFuncSetAttribute(tc_edge_kernel<false, F, W, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, es));
      DSB_CUDA_OK(cudaFuncSetAttribute(tc_edge_kernel<true, F, W, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, es));
      DSB_CUDA_OK(cudaFuncSetAttribute(tc_edge_kernel<true, F, W, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, es));
      DSB_CUDA_OK(cudaFuncSetAttribute(tc_edge_kernel<false, F, W, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, es));
      DSB_CUDA_OK(cudaFuncSetAttribute(tc_edge_kernel<false, F, W, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, es));
      DSB_CUDA_OK(cudaFuncSetAttribute(tc_edge_kernel<true, F, W, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, es));
      DSB_CUDA_OK(cudaFuncSetAttribute(tc_edge_kernel<true, F, W, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, es));
      return 0;
    });
    if (e) return e;
  }
  return 0;
}

int launch_tc_node_gemm(const dsb_dynamics* d, const GemmArgs& g, const TcImage& w, int n_tile_off, TcFormat fmt, int32_t* status,
                        cudaStream_t s) {
  (void)status;
  if (g.M == 0) return 0;
  const bool f16 = fmt != TcFormat::TF32x3;
  const int K = g.K1 + g.K2, TN = d->cfg.hidden_nf;
  if ((g.Nn % TN) || (K % TKC16) || (g.K1 % TKC16) || (g.lda1 % 4) || (g.ldc % 4)) {
    set_error("tc_node_gemm: unsupported shape K1=%d K2=%d Nn=%d", g.K1, g.K2, g.Nn);
    return DSB_ERR_INVALID_ARGUMENT;
  }
  TcGemmArgs a;
  a.A1 = g.A1; a.lda1 = g.lda1; a.K1 = g.K1; a.A2 = g.A2; a.lda2 = g.lda2; a.K2 = g.K2; a.div2 = g.div2; a.deg2 = g.deg2;
  const size_t img_off = (size_t)n_tile_off * (K / (f16 ? TKC16 : TKC)) * (size_t)(TN * TKC);     // skip the first n-tiles of the image
  a.Bhi = (f16 ? w.h_hi : w.t_hi) + img_off; a.Blo = (f16 ? w.h_lo : w.t_lo) + img_off;
  a.Z = g.Z; a.ldz = g.ldz;
  a.dead_nt = g.dead_cols / TN; a.dead_mt = a.dead_nt > 0 ? (g.dead_rows_from + TM - 1) / TM : 0;
  a.bias = g.bias; a.R = g.R; a.ldr = g.ldr; a.C = g.C; a.ldc = g.ldc; a.M = g.M; a.Nn = g.Nn; a.act = g.act;
  a.inv_scale = f16 ? w.h_inv : 1.0f;
  const int ntn_ = g.Nn / TN, ntm_ = (g.M + TM - 1) / TM;
  const int dmt_ = a.dead_nt > 0 ? (a.dead_mt < ntm_ ? a.dead_mt : ntm_) : ntm_;
  const int n_tiles = dmt_ * ntn_ + (ntm_ - dmt_) * (ntn_ - a.dead_nt);
  const int grid = n_tiles < d->num_sms ? n_tiles : d->num_sms;
  return dispatch_tc(fmt, TN, [&]<TcFormat F, int W>() -> int {
    DSB_CUDA_OK(launch_k(tc_node_gemm_kernel<F, W>, grid, TC_THREADS, gemm_smem_bytes<W>(), s, a));
    return 0;
  });
}

int launch_tc_edge_gcl(const dsb_dynamics* d, const Dims& dm, const Workspace& ws, const GclW& w, const float4* x, PView pv, TcFormat fmt,
                       int32_t* status, cudaStream_t s) {
  (void)status;
  const bool f16 = fmt != TcFormat::TF32x3;
  TcEdgeArgs a = {};
  a.P = pv.P; a.ldp = pv.ldp; a.x = x; a.cent = ws.cent; a.gid = ws.gid; a.vrow_ptr = ws.vrow_ptr; a.vmap = ws.vmap; a.n_rows = dm.N;
  a.erow = ws.erow; a.ecol = ws.ecol; a.ed0 = ws.ed0; a.NL = dm.NL; a.nm = 1;
  a.W2hi[0] = f16 ? w.iW2.h_hi : w.iW2.t_hi; a.W2lo[0] = f16 ? w.iW2.h_lo : w.iW2.t_lo;
  a.inv_scale[0] = f16 ? w.iW2.h_inv : 1.0f; a.inv_scale[1] = 1.0f;
  a.wr[0] = w.wr; a.wr0[0] = w.wr0; a.tb[0] = w.tb; a.b2[0] = w.b2;
  a.wa = w.wa; a.ba = w.ba; a.agg = ws.agg; a.part = ws.part; a.vcap = ws.vcap;
  const bool det = d->deterministic != 0;
  return dispatch_tc(fmt, d->cfg.hidden_nf, [&]<TcFormat F, int W>() -> int {
    auto kern = w.tb ? tc_edge_kernel<false, F, W, true> : tc_edge_kernel<false, F, W, false>;
    if (det) kern = w.tb ? tc_edge_kernel<false, F, W, true, true> : tc_edge_kernel<false, F, W, false, true>;
    DSB_CUDA_OK(launch_k(kern, d->num_sms, TC_THREADS, edge_smem_bytes<W>(), s, a));
    return 0;
  });
}

int launch_tc_edge_coord(const dsb_dynamics* d, const Dims& dm, const Workspace& ws, const EquivW& w, const float4* x, PView pv, TcFormat fmt,
                         int32_t* status, cudaStream_t s) {
  (void)status;
  const bool f16 = fmt != TcFormat::TF32x3;
  const dsb_config& c = d->cfg;
  TcEdgeArgs a = {};
  a.nm = c.reflection_equivariant ? 1 : 2;
  a.P = pv.P; a.ldp = pv.ldp; a.x = x; a.cent = ws.cent; a.gid = ws.gid; a.vrow_ptr = ws.vrow_ptr; a.vmap = ws.vmap; a.n_rows = dm.n_coord_rows;
  a.erow = ws.erow; a.ecol = ws.ecol; a.ed0 = ws.ed0; a.NL = dm.NL;
  a.inv_scale[0] = a.inv_scale[1] = 1.0f;
  for (int m = 0; m < a.nm; ++m) {
    a.W2hi[m] = f16 ? w.iW2[m].h_hi : w.iW2[m].t_hi; a.W2lo[m] = f16 ? w.iW2[m].h_lo : w.iW2[m].t_lo;
    a.inv_scale[m] = f16 ? w.iW2[m].h_inv : 1.0f;
    a.wr[m] = w.wr[m]; a.wr0[m] = w.wr0[m]; a.tb[m] = w.tb[m]; a.b2[m] = w.b2[m];
  }
  a.wa = w.w3; a.ba = nullptr;
  a.norm_constant = c.norm_constant; a.coords_range = c.coords_range; a.use_tanh = c.tanh; a.xagg = ws.xagg; a.part = ws.part; a.vcap = ws.vcap;
  const bool det = d->deterministic != 0;
  return dispatch_tc(fmt, c.hidden_nf, [&]<TcFormat F, int W>() -> int {
    auto kern = w.tb[0] ? tc_edge_kernel<true, F, W, true> : tc_edge_kernel<true, F, W, false>;
    if (det) kern = w.tb[0] ? tc_edge_kernel<true, F, W, true, true> : tc_edge_kernel<true, F, W, false, true>;
    DSB_CUDA_OK(launch_k(kern, d->num_sms, TC_THREADS, edge_smem_bytes<W>(), s, a));
    return 0;
  });
}

}  // namespace dsb
