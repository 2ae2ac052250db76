/*
 * diffsbdd_b200 — C ABI of the H100-native (sm_90a) DiffSBDD denoiser hot path.
 *
 * The reference has no FFI: its "plugin point" is the Python call
 *     EGNNDynamics.forward(xh_atoms, xh_residues, t, mask_atoms, mask_residues)
 * (reference equivariant_diffusion/dynamics.py:87-167) made once per DDPM step from
 * ConditionalDDPM.sample_p_zs_given_zt (conditional_model.py:445) and
 * EnVariationalDiffusion.sample_p_zs_given_zt (en_diffusion.py:503-557).
 * The entry points below are what a ctypes binding of that call needs: plain device pointers and
 * sizes, no torch types.  INTEGRATION.md shows the reference-side stub.
 *
 * All `const float*` / `float*` / `int64_t*` arguments are DEVICE pointers unless stated otherwise.
 * Every function returns 0 on success or a negative dsb_status; dsb_last_error() gives the text.
 * All kernels are launched on the caller's stream; no function synchronises the stream except
 * dsb_dynamics_create/destroy (weight packing) — forward is CUDA-graph capturable.
 */
#ifndef DIFFSBDD_B200_H_
#define DIFFSBDD_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  DSB_OK = 0,
  DSB_ERR_INVALID_ARGUMENT = -1,
  DSB_ERR_UNSUPPORTED_CONFIG = -2, /* mode 'gnn_dynamics', H not in {64..256 step 64}, tensor-core math modes with sin_embedding */
  DSB_ERR_CUDA = -3,
  DSB_ERR_WORKSPACE_TOO_SMALL = -4
} dsb_status;

/* Constructor arguments of EGNNDynamics (dynamics.py:11-19); same names, C types.
 * Cut-offs: a negative value means "None" (no cut-off for that block, dynamics.py:174-181). */
typedef struct {
  int32_t atom_nf;               /* dynamics.py:11 */
  int32_t residue_nf;
  int32_t n_dims;                /* must be 3 */
  int32_t joint_nf;
  int32_t hidden_nf;
  int32_t n_layers;
  int32_t inv_sublayers;
  int32_t attention;             /* bool */
  int32_t tanh;                  /* bool */
  int32_t condition_time;        /* bool */
  int32_t update_pocket_coords;  /* bool: joint model (dynamics.py:130-132, :161-164) */
  int32_t reflection_equivariant;/* bool: 0 -> cross-product MLP active (egnn_new.py:86-92) */
  int32_t edge_embedding_dim;    /* 0 = None (dynamics.py:51-53) */
  float norm_constant;           /* egnn_new.py:301, :315 */
  float normalization_factor;    /* egnn_new.py:327-328 ('sum' aggregation) */
  float coords_range;            /* 15.0: the undivided value the blocks receive (egnn_new.py:218) */
  float edge_cutoff_ligand;
  float edge_cutoff_pocket;
  float edge_cutoff_interaction;
  int32_t aggregation_mean;      /* bool: aggregation_method == 'mean' (egnn_new.py:330-334: sums divided by the receiver's edge count,
                                  * 1 for a receiver without edges) instead of 'sum' (divided by normalization_factor) */
  int32_t sin_embedding;         /* bool: the two squared distances of an edge enter the MLPs as 2 x 12 sinusoidal features
                                  * (egnn_new.py:282-293); fp32 FFMA kernels only (math mode 0) */
} dsb_config;

typedef struct dsb_dynamics dsb_dynamics; /* opaque: packed weights for one EGNNDynamics module */

/* ---- parameter table: the reference state-dict entries, in the order dsb_dynamics_create wants them.
 * Names are the reference's state_dict keys ("egnn.e_block_0.gcl_0.edge_mlp.0.weight", ...;
 * egnn_new.py:15-29, :78-92, :212-222; dynamics.py:27-53).  cross_product_mlp.4.weight is NOT listed:
 * it aliases coord_mlp.4.weight (egnn_new.py:78, :85, :91). */
int dsb_param_count(const dsb_config* cfg);
/* writes the NUL-terminated key of parameter i into buf; returns its element count, or <0. */
int64_t dsb_param_name(const dsb_config* cfg, int i, char* buf, size_t buflen);

/* ---- module lifetime.  `params[i]` is a device pointer to parameter i (fp32, contiguous, the
 * reference's own [out,in] layout).  The library copies/re-packs them into its own device buffer
 * (k-major GEMM operands, factorised first layers) — the caller's tensors are not referenced after
 * the call returns.  Replaces: EGNNDynamics.__init__ + load_state_dict (dynamics.py:11-85). */
int dsb_dynamics_create(const dsb_config* cfg, const float* const* params, int n_params,
                        dsb_dynamics** out);
void dsb_dynamics_destroy(dsb_dynamics* dyn);

/* Upper bound of directed edges incl. self loops for a batch: sum_g (n_lig_g + n_pocket_g)^2.
 * Host helper (host pointers). */
int64_t dsb_edge_capacity(const int64_t* n_lig_per_graph, const int64_t* n_pocket_per_graph,
                          int n_graphs);

/* Scratch the forward needs (activations, CSR edge list).  The caller owns the buffer (so that a
 * caching allocator / CUDA graph pool can provide it); contents need not be preserved between calls. */
size_t dsb_dynamics_workspace_bytes(const dsb_dynamics* dyn, int64_t n_atoms, int64_t n_residues,
                                    int64_t n_graphs, int64_t edge_capacity);

/* ---- the hot path.  Replaces EGNNDynamics.forward (dynamics.py:87-167), eval mode:
 *   xh_atoms    [n_atoms, 3+atom_nf]      xh_residues [n_residues, 3+residue_nf]   (row-major fp32)
 *   t           [t_numel]; t_numel == n_graphs (one per graph) or 1 (shared, dynamics.py:105-107)
 *   mask_atoms  [n_atoms] int64, mask_residues [n_residues] int64: non-decreasing graph ids in
 *               [0, n_graphs) (utils.py:146-154)
 *   out_atoms   [n_atoms, 3+atom_nf]      out_residues [n_residues, 3+residue_nf]
 *   status      device int32[4]: [0] |= 1 if a NaN reached the coordinate output (the reference raises
 *               ValueError("NaN detected in EGNN output"), dynamics.py:155-159 — the host wrapper
 *               turns the flag into that exception); [1] = number of edges of this call;
 *               [2] |= 1 if the edge list would not fit edge_capacity (outputs invalid); [3] reserved (always 0).
 *               Sticky: the library only ORs into [0] and [2]; the caller clears them.  (3xFP16 mode: an activation
 *               beyond the fp16 range becomes inf and reaches the output as NaN, i.e. flag [0].)
 * Inputs are not modified.  Asynchronous on `stream` (a cudaStream_t passed as void*). */
int dsb_dynamics_forward(dsb_dynamics* dyn,
                         const float* xh_atoms, const float* xh_residues,
                         const float* t, int64_t t_numel,
                         const int64_t* mask_atoms, const int64_t* mask_residues,
                         int64_t n_atoms, int64_t n_residues, int64_t n_graphs,
                         int64_t edge_capacity,
                         float* out_atoms, float* out_residues,
                         void* workspace, size_t workspace_bytes,
                         int32_t* status, void* stream);

/* ---- edge list only.  Replaces EGNNDynamics.get_edges (dynamics.py:169-187): same-graph pairs within
 * the per-block cut-offs, self loops kept, sorted by (row, col).  rows/cols: device int32[edge_capacity];
 * n_edges: device int32[1].  Uses `workspace` (same size contract as forward). */
int dsb_dynamics_edges(dsb_dynamics* dyn,
                       const float* xh_atoms, const float* xh_residues,
                       const int64_t* mask_atoms, const int64_t* mask_residues,
                       int64_t n_atoms, int64_t n_residues, int64_t n_graphs,
                       int64_t edge_capacity,
                       int32_t* rows, int32_t* cols, int32_t* n_edges,
                       void* workspace, size_t workspace_bytes, void* stream);

/* Number of kernel launches (memsets excluded) the last dsb_dynamics_forward on this module enqueued. */
int dsb_dynamics_last_launch_count(const dsb_dynamics* dyn);

/* ---- test hooks (host only; they change no kernel).  They let a test stop the forward after any operation and read its
 * workspace, so that every launch can be checked on its own against a float64 restatement of what it computes.
 *
 * dsb_dynamics_set_stop_after: afterwards dsb_dynamics_forward enqueues only its first n_ops operations (kernel launches
 * and memsets, counted in the fixed order the forward enqueues them) and returns 0.  A negative n_ops means no limit (the
 * default).  Returns the previous setting.  When the forward stops early, out_atoms / out_residues and status are not
 * written (except status[1] and [2] by the edge-list scan if it ran), and dsb_dynamics_last_launch_count counts the
 * launches that were enqueued.  Not for production use: a stopped forward computes nothing a caller can use. */
int dsb_dynamics_set_stop_after(dsb_dynamics* dyn, int n_ops);

/* dsb_workspace_region: byte offset and size of one region of the forward's workspace for the given config, mode
 * (deterministic 0/1) and sizes, as dsb_dynamics_forward lays it out.  The offset is from a workspace pointer aligned to
 * 256 bytes (the forward rounds the pointer it is given up to that alignment; caching allocators return such pointers).
 * N = n_atoms + n_residues, B = n_graphs, H = hidden_nf, nm = 2 without reflection equivariance, else 1:
 *   X_IN, X_PING, X_PONG  float4 [N + 1]  (x, y, z, 0) per node: input coordinates, then the blocks' outputs alternating
 *   H, HT, AGG            float [N + 1][H] (HT: N + 257 rows): node features, node-MLP hidden layer, raw receiver sums
 *   P                     float [N + 1][6 H]; the forward uses leading dimension (2 nm + 2) H: [coord/cross receiver |
 *                         coord/cross sender | next edge MLP receiver | sender] first-layer outputs
 *   XAGG, CENT, VELMEAN   float4 [N + 1], [B + 1], [B + 1]: raw coordinate sums, per-graph centroids, velocity means
 *   DEG, ROW_PTR, VROW_PTR int32 [N + 1], [N + 2], [N + 2];  VMAP int32 [edge_capacity + 3 N + 1]
 *   EROW, ECOL, ED0       int32 / int32 / float [edge_capacity + 1]: CSR edges and their input-geometry d^2
 *   PART                  deterministic mode only (0 bytes otherwise): per-chunk partial sums
 *   LIG_OFF, POC_OFF, GID int32 [B + 2], [B + 2], [N + 1]
 * Returns 0, or a negative dsb_status for a bad config, size or region. */
enum {
  DSB_WS_X_IN = 0, DSB_WS_X_PING, DSB_WS_X_PONG, DSB_WS_H, DSB_WS_HT, DSB_WS_AGG, DSB_WS_P, DSB_WS_XAGG, DSB_WS_CENT,
  DSB_WS_DEG, DSB_WS_ROW_PTR, DSB_WS_VROW_PTR, DSB_WS_VMAP, DSB_WS_EROW, DSB_WS_ECOL, DSB_WS_ED0, DSB_WS_PART,
  DSB_WS_LIG_OFF, DSB_WS_POC_OFF, DSB_WS_GID, DSB_WS_VELMEAN, DSB_WS_REGIONS
};
int dsb_workspace_region(const dsb_config* cfg, int deterministic, int64_t n_atoms, int64_t n_residues, int64_t n_graphs,
                         int64_t edge_capacity, int region, int64_t* offset, int64_t* bytes);

/* Process-wide switch for programmatic dependent launch of the forward's kernels (each kernel's launch and prologue
 * overlap its predecessor's tail; every kernel executes griddepcontrol.wait before touching data a predecessor may
 * have written).  enable: 1 on, 0 off, negative = query only.  Returns the previous setting.  Initial value: the
 * environment variable DSB_PDL (default on).  No effect on results. */
int dsb_set_programmatic_launch(int enable);

/* ---- arithmetic path.  mode is a bitmask: 1 = node GEMMs, 2 = edge (GCL) kernel, 4 = coordinate edge kernel run on
 * the tensor pipe (wgmma, accumulators in registers) as 3-product split contractions with fp32 accumulation
 * (x.w ~= x_lo.w_hi + x_hi.w_lo + x_hi.w_hi: fp32-grade accuracy, inside the atol 1e-5 / rtol 1e-4 parity tolerance);
 * 8 selects the operand format of those kernels: 0 = 3xTF32 (tf32 operands, 8-bit exponent, any range),
 * 8 = 3xFP16 (f16 operands: half the shared-memory operand traffic, twice the MMA rate; weights are pre-scaled per matrix
 * with an exact power of two; an activation beyond the fp16 range turns into NaN at the output and raises through
 * status[0]).  16, valid only together with 8, = single product: x.w ~= x_hi.w_hi, the fp16 operands of the 3xFP16 split
 * without their residuals, accumulated in fp32 (a third of the wgmmas, half the operand stores and weight-stream bytes).
 * Its accuracy is fp16-grade, not fp32-grade: each operand carries a relative rounding error up to 2^-11, so a contraction
 * is off by up to ~2^-10 sum|x||w| and results are well outside the fp32 parity tolerance; its range limit is that of
 * 3xFP16.  Bit 16 without bit 8 returns DSB_ERR_INVALID_ARGUMENT.  0 = fp32 FFMA kernels everywhere.  Only hidden_nf
 * 128, 192 and 256 have tensor-core kernels. */
int dsb_dynamics_set_math_mode(dsb_dynamics* dyn, int mode);

/* ---- deterministic mode (per module; default off).  enable: 1 on, 0 off, negative = query only.  Returns the previous
 * setting (0 or 1), or DSB_ERR_INVALID_ARGUMENT for a NULL module.
 * Off: every receiver sum of the edge kernels (GCL aggregate, coordinate update) is accumulated with floating-point
 * atomics, whose order depends on timing; a receiver with more than two such contributions can differ in its last bits
 * from run to run.
 * On: the edge kernels store per-chunk partial sums (4 rows of one receiver in the padded edge order, in row order) and
 * one extra kernel per edge launch sums each receiver's chunks in ascending order.  The summation order of every
 * receiver's sum is then a function of that receiver's own edges, so dsb_dynamics_forward gives bit-identical outputs
 * for bit-identical inputs (the whole batch: every graph, in the same order), weights and math mode on the same GPU
 * model with the same library build, independent of the run or process, eager launch vs. CUDA-graph replay,
 * programmatic dependent launch, workspace / output addresses and the persistent grid size.  A graph's outputs also do
 * not depend bitwise on the other graphs of the batch, in any math mode: the same graph denoised alone or inside any
 * batch, at any position, gives the same bits (the tensor-core edge kernels' shared-reciprocal SiLU groups values of one
 * edge only in this mode), so one graph can be regenerated on its own.  Results are not bit-identical
 * across math modes, nor with the default mode.  If the edges of a call exceed edge_capacity (status[2]) the outputs are
 * invalid as in the default mode; the deterministic kernels then stop at the end of the partial buffer.  Cost: dsb_dynamics_workspace_bytes grows by a partial buffer of
 * ceil((edge_capacity + 3 (n_atoms + n_residues)) / 128) * 32 * hidden_nf floats, and dsb_dynamics_forward enqueues one
 * more kernel per GCL sub-layer and per coordinate update (dsb_dynamics_last_launch_count counts them).  Status-flag
 * semantics are unchanged.  Call it outside stream capture: a captured forward keeps the mode it was captured in. */
int dsb_dynamics_set_deterministic(dsb_dynamics* dyn, int enable);

/* ---- measurement hook (bench.py's live roofline).  When enabled, every non-captured forward brackets
 * its launches with CUDA events on the launch stream, grouped into 7 kernel classes:
 *   0 setup (plan, encoders+embedding, edge list)  1 node GEMMs  2 memsets  3 edge_gcl_kernel
 *   4 edge_coord_kernel  5 coord finish/centroid  6 decoders/output.
 * collect() synchronises the recorded events and returns accumulated milliseconds and interval counts per
 * class (host arrays of 7); reset != 0 clears the accumulators. */
int dsb_dynamics_set_profiling(dsb_dynamics* dyn, int enabled);
int dsb_dynamics_collect_profile(dsb_dynamics* dyn, double* ms_by_class, int64_t* count_by_class, int reset);

/* ---- fused DDPM ligand update (one launch). Replaces the element-wise tail of
 * ConditionalDDPM.sample_p_zs_given_zt (conditional_model.py:451-460) + sample_normal_zero_com
 * (:140-160) + remove_mean_batch (:688-696):
 *   mu   = z/alpha_ts[g] - coef1[g] * eps_hat
 *   z'   = mu + sigma[g] * noise ;   com_g = mean over ligand atoms of graph g of z'[:, :3]
 *   z_out[:, :3] = z'[:, :3] - com_g ; z_out[:, 3:] = z'[:, 3:]
 *   pocket_out[:, :3] = pocket[:, :3] - com_g ; pocket_out[:, 3:] = pocket[:, 3:]
 * coef: device fp32 [n_graphs, 3] = (alpha_ts, sigma2_ts/alpha_ts/sigma_t, sigma) per graph (z is DIVIDED by
 * alpha_ts, exactly as conditional_model.py:451 does).
 * In-place allowed (z_out == z, pocket_out == pocket). */
int dsb_ddpm_ligand_update(const float* z_lig, const float* eps_hat, const float* noise,
                           const float* coef, const int64_t* mask_atoms, const int64_t* mask_residues,
                           const float* xh_pocket, int64_t n_atoms, int64_t n_residues,
                           int64_t n_graphs, int32_t atom_nf, int32_t residue_nf,
                           float* z_out, float* xh_pocket_out, void* stream);

/* ---- fused RePaint iteration of ConditionalDDPM.inpaint (one launch; conditional_model.py:636-666), run right after
 * dsb_ddpm_ligand_update, in place on its outputs (z_lig = z_unknown, xh_pocket):
 *   xk      = xh_known, coordinates shifted by (COM(pocket) - com_pocket0[g])                         (:636-640)
 *   z_known = alpha_s xk + sigma_s noise_known ; ligand COM of z_known removed from z_known and pocket   (:162-183)
 *   dx      = COM_fixed(z_unknown) - COM_fixed(z_known) ; z_known.x += dx ; pocket.x += dx               (:645-656)
 *   z       = z_known * fixed + z_unknown * (1 - fixed)                                                  (:659)
 *   if noise_renoise != NULL:  z = alpha_ts z + sigma_ts noise_renoise, ligand COM removed from z and pocket  (:420-430, :662-666)
 * xh_known [n_atoms, 3+atom_nf] (normalised known ligand), com_pocket0 [n_graphs, 3] (pocket COM before sampling),
 * lig_fixed [n_atoms] (0/1 as fp32), coef [n_graphs, 4] = (alpha_s, sigma_s, alpha_{t|s}, sigma_{t|s}). */
int dsb_ddpm_inpaint_update(float* z_lig, float* xh_pocket, const float* xh_known, const float* com_pocket0,
                            const float* lig_fixed, const float* noise_known, const float* noise_renoise,
                            const float* coef, const int64_t* mask_atoms, const int64_t* mask_residues,
                            int64_t n_atoms, int64_t n_residues, int64_t n_graphs, int32_t atom_nf,
                            int32_t residue_nf, void* stream);

/* ---- joint model (EnVariationalDiffusion, update_pocket_coords = 1): the same two fusions for ligand AND pocket.
 * noise_x is ONE tensor [n_atoms + n_residues, 3] (ligand rows first) as sample_center_gravity_zero_gaussian_batch draws it
 * (en_diffusion.py:559-578); its per-graph mean over ligand+pocket nodes is removed inside the kernel (:940-944).
 * dsb_ddpm_joint_update  = tail of EnVariationalDiffusion.sample_p_zs_given_zt (en_diffusion.py:540-557):
 *   z' = z/alpha_ts - coef1 * eps_hat + sigma * eps ; joint COM of z'.x removed.  coef [n_graphs, 3] as dsb_ddpm_ligand_update.
 * dsb_ddpm_joint_inpaint_update = one RePaint iteration of EnVariationalDiffusion.inpaint after that step (:741-807):
 *   z_known = alpha_s xh0 + sigma_s eps ; COM of the fixed nodes aligned noised -> denoised ; blend by lig_fixed / pocket_fixed ;
 *   if renoise_x != NULL: jump back z = alpha_{t|s} z + sigma_{t|s} eps' with the joint COM removed (sample_p_zt_given_zs).
 *   coef [n_graphs, 4] = (alpha_s, sigma_s, alpha_{t|s}, sigma_{t|s}); xh0_* = known data, normalised and centred as :707-717. */
int dsb_ddpm_joint_update(float* z_lig, float* z_pocket, const float* eps_lig, const float* eps_pocket,
                          const float* noise_x, const float* noise_h_lig, const float* noise_h_pocket,
                          const float* coef, const int64_t* mask_atoms, const int64_t* mask_residues,
                          int64_t n_atoms, int64_t n_residues, int64_t n_graphs, int32_t atom_nf,
                          int32_t residue_nf, void* stream);
int dsb_ddpm_joint_inpaint_update(float* z_lig, float* z_pocket, const float* xh0_lig, const float* xh0_pocket,
                                  const float* lig_fixed, const float* pocket_fixed, const float* noise_x,
                                  const float* noise_h_lig, const float* noise_h_pocket, const float* renoise_x,
                                  const float* renoise_h_lig, const float* renoise_h_pocket, const float* coef,
                                  const int64_t* mask_atoms, const int64_t* mask_residues, int64_t n_atoms,
                                  int64_t n_residues, int64_t n_graphs, int32_t atom_nf, int32_t residue_nf,
                                  void* stream);

/* ---- DPM-Solver++(2M) step in data-prediction form (one launch, one block per graph; DESIGN §13), both models:
 *   x0 = (z - sigma_t[g] eps_hat) * inv_alpha_t[g]                      (prediction of the clean sample)
 *   D  = (1 + w[g]) x0 - w[g] hist ; D = x0 when w[g] == 0 (first step: hist is not read)
 *   z' = c0[g] z + c1[g] D ;  hist' = x0
 * then the COM of z'.x is removed from z'.x, from the pocket coordinates and from hist'.x:
 *   joint == 0 (ConditionalDDPM): the LIGAND COM; the pocket (z_pocket) is only shifted; hist_pocket and eps_pocket are
 *                                 not used and may be NULL.
 *   joint != 0 (EnVariationalDiffusion): ligand AND pocket are updated and the COM is taken over ligand + pocket nodes.
 * coef: device fp32 [n_graphs, 5] = (sigma_s/sigma_t, -alpha_s (e^-h - 1), 1/alpha_t, sigma_t, w) with h = lambda_s - lambda_t,
 * lambda = -gamma/2, w = h / (2 h_prev) (0 on the first step).  hist_* [rows, 3 + nf]: x0 of the previous step in the current
 * frame.  In place on z_lig, z_pocket, hist_lig, hist_pocket.  Masks sorted; each graph's sums run in a fixed order without
 * atomics, so the result repeats bit for bit and a graph's result does not depend on the rest of its batch. */
int dsb_ddpm_multistep_update(float* z_lig, float* z_pocket, float* hist_lig, float* hist_pocket, const float* eps_lig,
                              const float* eps_pocket, const float* coef, const int64_t* mask_atoms,
                              const int64_t* mask_residues, int64_t n_atoms, int64_t n_residues, int64_t n_graphs,
                              int32_t atom_nf, int32_t residue_nf, int32_t joint, void* stream);

/* ---- RePaint round with the DPM-Solver++(2M) step (one launch, one block per graph; DESIGN §14), both models.  On entry z is
 * z_t of the round; per graph, in place:
 *   1. the 2M step of dsb_ddpm_multistep_update: x0 = (z - sigma_t eps_hat) * inv_alpha_t ; D = (1 + w) x0 - w hist (x0 when
 *      w == 0) ; z' = c0 z + c1 D ; the COM of z'.x removed (joint == 0: ligand COM from z', the pocket and hist ;
 *      joint != 0: ligand + pocket COM from z' and hist of both).
 *   2. the RePaint iteration on z' as the unknown part:
 *      joint == 0: dsb_ddpm_inpaint_update with (known_lig, com_pocket0, lig_fixed, noise_known, renoise); known_pocket,
 *                  pocket_fixed, eps_pocket, hist_pocket and the *_h_* noises are not used and may be NULL.
 *      joint != 0: dsb_ddpm_joint_inpaint_update with (known_lig, known_pocket, lig_fixed, pocket_fixed, noise_known +
 *                  noise_known_h_*, renoise + renoise_h_*); com_pocket0 is not used and may be NULL.
 *      renoise == NULL: no re-noising (the round that ends a grid step).
 * hist_* [rows, 3 + nf]: x0 of the previous grid step, in the frame of the pocket (joint == 0) or of z (joint != 0).  Every
 * translation the round applies to the pocket coordinates (joint == 0: the 2M COM removal, the known part's COM removal, the
 * fixed-COM shift, the re-noise COM removal) or to z (joint != 0: the 2M and the re-noise COM removals) is applied to hist.x as
 * well.  commit != 0: x0 of this round replaces the history before those translations; commit == 0: the history is only
 * translated.
 * coef: device fp32 [n_graphs, 9] = (sigma_s/sigma_t, -alpha_s (e^-h - 1), 1/alpha_t, sigma_t, w) as dsb_ddpm_multistep_update,
 * then (alpha_s, sigma_s, alpha_{t|s}, sigma_{t|s}) as the RePaint entries.  Noise layouts as dsb_ddpm_inpaint_update
 * (joint == 0: [n_atoms, 3 + atom_nf]) and dsb_ddpm_joint_inpaint_update (joint != 0: x [n_atoms + n_residues, 3], h per part).
 * Masks sorted; each graph's sums run in a fixed order without atomics, so the result repeats bit for bit and a graph's result
 * does not depend on the rest of its batch. */
int dsb_ddpm_multistep_inpaint_update(float* z_lig, float* z_pocket, float* hist_lig, float* hist_pocket, const float* eps_lig,
                                      const float* eps_pocket, const float* known_lig, const float* known_pocket,
                                      const float* com_pocket0, const float* lig_fixed, const float* pocket_fixed,
                                      const float* noise_known, const float* noise_known_h_lig, const float* noise_known_h_pocket,
                                      const float* renoise, const float* renoise_h_lig, const float* renoise_h_pocket,
                                      const float* coef, const int64_t* mask_atoms, const int64_t* mask_residues, int64_t n_atoms,
                                      int64_t n_residues, int64_t n_graphs, int32_t atom_nf, int32_t residue_nf, int32_t joint,
                                      int32_t commit, void* stream);

/* ---- DPM-Solver++(3M) step in data-prediction form (one launch, one block per graph; DESIGN §15), both models:
 *   x0 = (z - sigma_t[g] eps_hat) * inv_alpha_t[g]
 *   z' = c0[g] z + k0[g] x0 + k1[g] m1 + k2[g] m2 ; m1 = hist is read only when k1[g] != 0, m2 = hist2 only when k2[g] != 0
 *   hist2' = m1 (x0 when k1[g] == 0) ; hist' = x0
 * then the COM of z'.x is removed from z'.x, from the pocket coordinates and from hist'.x and hist2'.x, as in
 * dsb_ddpm_multistep_update (joint == 0: the LIGAND COM, the pocket only shifted, hist_pocket, hist2_pocket and eps_pocket not
 * used and may be NULL; joint != 0: ligand AND pocket updated, COM over ligand + pocket nodes).
 * coef: device fp32 [n_graphs, 6] = (sigma_s/sigma_t, 1/alpha_t, sigma_t, k0, k1, k2): en_diffusion.fast_coefficients
 * ('dpmpp_3m'), with k1 = k2 = 0 on the first step run and k2 = 0 on the second.  hist_* / hist2_* [rows, 3 + nf]: x0 of the
 * previous step and of the one before it, in the current frame.  In place on z_*, hist_*, hist2_*.  Masks sorted; each graph's
 * sums run in a fixed order without atomics, so the result repeats bit for bit and a graph's result does not depend on the rest
 * of its batch. */
int dsb_ddpm_multistep3_update(float* z_lig, float* z_pocket, float* hist_lig, float* hist_pocket, float* hist2_lig,
                               float* hist2_pocket, const float* eps_lig, const float* eps_pocket, const float* coef,
                               const int64_t* mask_atoms, const int64_t* mask_residues, int64_t n_atoms, int64_t n_residues,
                               int64_t n_graphs, int32_t atom_nf, int32_t residue_nf, int32_t joint, void* stream);

/* ---- RePaint round with the DPM-Solver++(3M) step (one launch, one block per graph; DESIGN §15), both models: as
 * dsb_ddpm_multistep_inpaint_update with the 3M step of dsb_ddpm_multistep3_update in place of the 2M step.  Every translation
 * the round applies to hist.x is applied to hist2.x too.  commit != 0: hist2 <- hist (x0 when k1 == 0) and hist <- x0 before
 * those translations; commit == 0: both histories are only translated.
 * coef: device fp32 [n_graphs, 10] = the 3M row (6) of dsb_ddpm_multistep3_update, then (alpha_s, sigma_s, alpha_{t|s},
 * sigma_{t|s}) as the RePaint entries.  Pointers that a model does not use may be NULL as in
 * dsb_ddpm_multistep_inpaint_update (hist2_pocket with hist_pocket). */
int dsb_ddpm_multistep3_inpaint_update(float* z_lig, float* z_pocket, float* hist_lig, float* hist_pocket, float* hist2_lig,
                                       float* hist2_pocket, const float* eps_lig, const float* eps_pocket, const float* known_lig,
                                       const float* known_pocket, const float* com_pocket0, const float* lig_fixed,
                                       const float* pocket_fixed, const float* noise_known, const float* noise_known_h_lig,
                                       const float* noise_known_h_pocket, const float* renoise, const float* renoise_h_lig,
                                       const float* renoise_h_pocket, const float* coef, const int64_t* mask_atoms,
                                       const int64_t* mask_residues, int64_t n_atoms, int64_t n_residues, int64_t n_graphs,
                                       int32_t atom_nf, int32_t residue_nf, int32_t joint, int32_t commit, void* stream);

/* ---- evaluation-mode variational bound (validation / test NLL): what EnVariationalDiffusion.forward, ConditionalDDPM.forward
 * and SimpleConditionalDDPM.forward compute in eval mode besides the two denoiser calls and the per-graph scalar algebra.
 *
 * dsb_ddpm_noise = q(z_t | x, h) without a COM projection (en_diffusion.py:302-317; SimpleConditionalDDPM, conditional_model.py:702-735):
 *   z_lig = alpha[g] xh_lig + sigma[g] eps_lig ;  z_pocket = alpha[g] xh_pocket + sigma[g] eps_pocket (skipped if xh_pocket == NULL).
 * coef [n_graphs, 2] = (alpha_t, sigma_t).  For the joint model eps.x must already be COM-free over ligand + pocket.
 * (ConditionalDDPM noises with dsb_ddpm_ligand_update and coef = (1/alpha_t, 0, sigma_t): z = xh/(1/alpha) + sigma eps, ligand COM
 * removed from z and pocket, conditional_model.py:162-183.)
 *
 * dsb_ddpm_vlb_terms: one block per graph over the row ranges of the sorted masks, fixed summation order (no atomics), so `terms`
 * repeats bit for bit for identical inputs.  Inputs [rows, 3+nf] fp32:
 *   xh0_*   the normalised data x (as noised) | h = (one_hot - norm_bias_h) / norm_value_h ; its h columns are the one-hot
 *   z_t_lig, eps_t_*, net_t_*   noised sample, noise and denoiser output at the random t
 *   z_0_*,   eps_0_*, net_0_*   the same at t = 0
 * The pocket pointers are all NULL for the conditional models (ligand-only likelihood).
 * coef [n_graphs, 4] = (alpha_T, sigma_0 * norm_value_h, alpha_t, sigma_t).  vnode_idx: ligand class of virtual atoms (-1 = none);
 * the x columns of ligand rows whose h column vnode_idx is non-zero are left out of columns 0 and 2 (conditional_model.py:76-78).
 * terms [n_graphs, DSB_VLB_TERMS], per graph:
 *   0 sum (eps_t - net_t)^2 ligand (all columns)         1 the same, pocket                     -> error_t (:262-267, en_diffusion.py:385-390)
 *   2 sum (eps_0.x - net_0.x)^2 ligand                   3 the same, pocket                     -> -2 log p(x | z_0) w/o constants
 *   4 log p(h | z_0), ligand + pocket: sum over nodes of one_hot . (log(Phi((c+1/2)/s0) - Phi((c-1/2)/s0) + 1e-10) - logsumexp),
 *     c = z_0.h * norm_value_h + norm_bias_h - 1, Phi(x) = (1 + erf(x / sqrt 2)) / 2, one_hot un-normalised (en_diffusion.py:185-261)
 *   5 |alpha_T x|^2, ligand + pocket   6 |alpha_T h|^2, ligand + pocket                          -> kl_prior (en_diffusion.py:109-155)
 *   7 sum |net_t.x| ligand   8 sum |net_t.h| ligand   9 sum |net_t.x| pocket   10 sum |net_t.h| pocket  -> the info means (:451-464)
 * xh_lig_hat [n_atoms, 3+atom_nf] = z_t / alpha_t - net_t * sigma_t / alpha_t (en_diffusion.py:471-477). */
#define DSB_VLB_TERMS 11
int dsb_ddpm_noise(const float* xh_lig, const float* eps_lig, const float* xh_pocket, const float* eps_pocket,
                   const float* coef, const int64_t* mask_atoms, const int64_t* mask_residues, int64_t n_atoms,
                   int64_t n_residues, int64_t n_graphs, int32_t atom_nf, int32_t residue_nf, float* z_lig, float* z_pocket,
                   void* stream);
int dsb_ddpm_vlb_terms(const float* xh0_lig, const float* z_t_lig, const float* eps_t_lig, const float* net_t_lig,
                       const float* z_0_lig, const float* eps_0_lig, const float* net_0_lig, const float* xh0_pocket,
                       const float* eps_t_pocket, const float* net_t_pocket, const float* z_0_pocket, const float* eps_0_pocket,
                       const float* net_0_pocket, const float* coef, const int64_t* mask_atoms, const int64_t* mask_residues,
                       int64_t n_atoms, int64_t n_residues, int64_t n_graphs, int32_t atom_nf, int32_t residue_nf,
                       float norm_value_h, float norm_bias_h, int32_t vnode_idx, float* terms, float* xh_lig_hat, void* stream);

/* ---- seeded per-graph random numbers (the samplers' `seeds=` argument).  Fills out [rows, cols] (row-major fp32) so that a
 * value depends only on (seed of its graph, draw id, role, row index within its graph, column), never on the other graphs
 * of the batch or on the row's position in it.  This mapping is a reproducibility contract: a sampled ligand is a function
 * of its seed, so changing any step below changes every seeded result.
 *   role  DSB_RNG_LIGAND:  rows = n_atoms, graph g = mask_atoms[r], index i = r - (first row of g)
 *         DSB_RNG_POCKET:  rows = n_residues over mask_residues, likewise
 *         DSB_RNG_JOINT_X: rows = n_atoms + n_residues (ligand rows first, as the joint model's shared coordinate noise);
 *                          a pocket row's index is (ligand rows of g) + its index among g's pocket rows
 *         DSB_RNG_GRAPH:   rows = n_graphs, g = r, i = 0 (one row per graph, e.g. the size prior)
 *   key      (k0, k1) = (low, high) 32-bit words of seeds[g] (int64, device)
 *   counter  (c0, c1, c2, c3) = (column group j = col / 4, i, role | (draw >> 32) << 4, draw & 0xffffffff), draw = *draw_id
 *            (int64, device: read at run time, so one captured graph serves every step)
 *   words    (w0, w1, w2, w3) = Philox4x32-10(counter, key) (Random123 constants; the key is bumped after every round)
 *   kind DSB_RNG_NORMAL:  U(w) = fmaf((float)w, 2^-32, 2^-33) in (0, 1] ((float)w rounds to nearest);
 *                         columns 4j, 4j+1 = r0 cos(2 pi v0), r0 sin(2 pi v0) with r0 = sqrtf(-2 logf(U(w0))),
 *                         v0 = (float)w1 * 2^-32 (sincospif(2 v0)); columns 4j+2, 4j+3 the same from (w2, w3)
 *        DSB_RNG_UNIFORM: columns 4j+k = U(wk) in (0, 1]
 *        DSB_RNG_BITS:    columns 4j+k = the raw word wk (bit pattern stored in the fp32 slot)
 * Columns past `cols` of the last group are dropped.  Capturable; touches no other generator state. */
enum { DSB_RNG_LIGAND = 0, DSB_RNG_POCKET = 1, DSB_RNG_JOINT_X = 2, DSB_RNG_GRAPH = 3 };
enum { DSB_RNG_NORMAL = 0, DSB_RNG_UNIFORM = 1, DSB_RNG_BITS = 2 };
int dsb_seeded_normal(float* out, int64_t cols, int32_t role, int32_t kind, const int64_t* seeds, const int64_t* draw_id,
                      const int64_t* mask_atoms, const int64_t* mask_residues, int64_t n_atoms, int64_t n_residues,
                      int64_t n_graphs, void* stream);

const char* dsb_last_error(void);
const char* dsb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* DIFFSBDD_B200_H_ */
