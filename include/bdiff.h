/*
 * bdiff.h — C ABI of libbdiff_sm90.so: the H100-native GCPNet denoiser hot path of GCDM.
 *
 * The reference (BioinfoMachineLearning/bio-diffusion) has no FFI for this path; its seam is the Python
 * class contract `dynamics_network.forward(batch, xh, t) -> (batch, net_out)` selected in
 * src/models/qm9_mol_gen_ddpm.py:101-105,125-131 (and geom_mol_gen_ddpm.py) and called from
 * src/models/components/variational_diffusion.py:873,1042,1116,1236.  The entry points below are what a
 * binding for that seam needs; each cites the reference interface it replaces.  Host mirror:
 * bio-diffusion_b200/bdiff/dynamics.py (class GCPNetDynamicsB200); binding recipe: INTEGRATION.md.
 *
 * Conventions
 *   - plain C, no torch types; every data pointer is a DEVICE pointer owned by the caller unless the name
 *     ends in _host; float = fp32, indices int64 at the boundary (like the reference), mask = uint8 (0/1);
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream); nothing synchronises the
 *     device except bdiff_plan_topology (one D2H of batch_index/mask + one H2D of the plan);
 *   - return 0 on success, a negative BDIFF_E* code otherwise; never throws; bdiff_last_error(h) gives text;
 *   - one handle per (device, stream); not thread-safe; the handle owns packed weights and workspace.
 */
#ifndef BDIFF_H_
#define BDIFF_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BDIFF_OK 0
#define BDIFF_EINVAL (-1)   /* bad argument / unsupported configuration            */
#define BDIFF_ECUDA (-2)    /* a CUDA runtime call or kernel launch failed         */
#define BDIFF_ESTATE (-3)   /* call order violated (weights missing, no plan, ...) */
#define BDIFF_ENOMEM (-4)

#define BDIFF_ABI_VERSION 1

#if defined(__GNUC__)
#define BDIFF_API __attribute__((visibility("default")))
#else
#define BDIFF_API
#endif

/* Compute modes.  PARITY: every multiply-add in fp32 FFMA (differs from the reference only by
 * summation order).  TENSOR: the dense GEMMs of the layers run on the tensor cores (wgmma) with split-bf16
 * operands and fp32 accumulation. */
#define BDIFF_MODE_PARITY_FP32 0
#define BDIFF_MODE_TENSOR 1

typedef struct bdiff_handle bdiff_handle;

/* Dims of the denoiser; mirrors what GCPNetDynamics.__init__ derives from its five Hydra configs
 * (src/models/components/gcpnet.py:933-1039).  Only the shipped option set is supported (GCP2,
 * vector_gate, no frame_gate, bottleneck 4, 4 residual message GCPs, scalar message attention, one
 * feed-forward GCP, no GCP norm / dropout, no self-conditioning); anything else -> BDIFF_EINVAL. */
typedef struct bdiff_config {
  int32_t num_h;          /* F: node scalar features in xh = [x(3) | h(F)] = num_atom_types + include_charges */
  int32_t num_context;    /* len(module_cfg.conditioning): context columns appended after the time column     */
  int32_t num_layers;     /* model_cfg.num_encoder_layers (9 QM9, 4 GEOM)                                      */
  int32_t h_hidden;       /* model_cfg.h_hidden_dim   — must be 256                                            */
  int32_t chi_hidden;     /* model_cfg.chi_hidden_dim — must be 32                                             */
  int32_t e_hidden;       /* model_cfg.e_hidden_dim   (64 QM9, 16 GEOM), multiple of 4, <= 64                   */
  int32_t xi_hidden;      /* model_cfg.xi_hidden_dim  (16 QM9, 8 GEOM), multiple of 4, <= 16                    */
  int32_t mode;           /* BDIFF_MODE_*                                                                       */
} bdiff_config;

BDIFF_API int32_t bdiff_abi_version(void);

/* Replaces: GCPNetDynamics.__init__ (gcpnet.py:933-1039) — allocates packed-weight storage. */
BDIFF_API int32_t bdiff_create(const bdiff_config* cfg, bdiff_handle** out);
BDIFF_API void bdiff_destroy(bdiff_handle* h);
BDIFF_API const char* bdiff_last_error(const bdiff_handle* h);   /* h may be NULL: last creation error */

/* Replaces: nn.Module.load_state_dict on the reference module.  `name` is the reference parameter name
 * relative to the denoiser (e.g. "interaction_layers.3.interaction.message_fusion.0.scalar_out.weight"),
 * `data` a contiguous fp32 device tensor of `shape`.  The tensor is repacked (transposed to K-major,
 * split, zero-padded) into the kernel layout immediately on `stream`; the caller may free it afterwards. */
BDIFF_API int32_t bdiff_set_weight(bdiff_handle* h, void* stream, const char* name, const float* data,
                         const int64_t* shape, int32_t ndim);
/* Number of reference parameter tensors still missing (0 = ready); -errno on error. */
BDIFF_API int32_t bdiff_weights_missing(const bdiff_handle* h);

/* Finishes weight preparation once every parameter is set (tensor mode: builds the pre-swizzled bf16 weight
 * K-blocks the TMA producer streams).  Called by the host after load_state_dict so that nothing but the forward
 * kernels runs inside a captured CUDA graph.  Idempotent. */
BDIFF_API int32_t bdiff_prepare(bdiff_handle* h, void* stream);

/* Hardware self test of the split-bf16 machinery of the tensor mode (csrc/bdiff_selftest.cu): hi/lo A blocks,
 * un-swizzled K=16 weight slabs, three (variant bit 1: four, node-tile row views) products per K step, accumulator
 * scratch pair exchange.  C[128,336] <- [A W^T (320 cols; the last 32 negated) | exchange (16 cols)] for
 * A fp32[128,128], W fp32[320,128] (device pointers).  Synchronises. */
BDIFF_API int32_t bdiff_selftest_split(void* stream, int32_t variant, const float* A, const float* W, float* C);


/* Replaces: GCPNetDynamics.get_fully_connected_edge_index (gcpnet.py:1054-1066) — as an implicit plan.
 * batch_index int64[N] (sorted molecule ids, as every caller provides), mask uint8[N].  Builds the
 * per-molecule offsets the kernels enumerate edges from; *num_edges_host receives E = sum_k nact_k^2.
 * Synchronises `stream` (one small D2H + H2D).  Re-plan whenever batch_index / mask change. */
BDIFF_API int32_t bdiff_plan_topology(bdiff_handle* h, void* stream, int32_t num_mols, int64_t num_nodes,
                            const int64_t* batch_index, const uint8_t* mask, int64_t* num_edges_host);

/* Materialises the reference's edge_index int64[2,E] ((row,col)-sorted, self loops, masked nodes dropped)
 * from the current plan — only for callers/tests that want it; the kernels never read it. */
BDIFF_API int32_t bdiff_edge_index(bdiff_handle* h, void* stream, int64_t* edge_index);

/* Replaces: GCPNetDynamics.forward / atom_types_and_coords_forward (gcpnet.py:1042-1052, 1069-1232).
 * xh fp32[N,3+F], t fp32[N] (per node, the reference's t[batch_index]), context fp32[N,C] or NULL,
 * net_out fp32[N,3+F] = [vel (CoG-free) | h_final].  xh is not modified. */
BDIFF_API int32_t bdiff_denoise_forward(bdiff_handle* h, void* stream, const float* xh, const float* t,
                              const float* context, float* net_out);

/* Same as bdiff_denoise_forward, but records CUDA events on `stream` around every kernel class and, after
 * synchronising the stream, writes milliseconds to ms_host[0..6] = {prep+node_frames, edge_embed, node_embed,
 * edge_message (sum over layers), node_update (sum over layers), finalize, whole forward}; ms_host[7] = number
 * of edge_message launches.  Measurement hook for bench.py's roofline block (not on the product path). */
BDIFF_API int32_t bdiff_profile_forward(bdiff_handle* h, void* stream, const float* xh, const float* t,
                                        const float* context, float* net_out, float* ms_host);

/* Optional taps of the last forward, for parity tests: which = "f_ij" [E,9], "e" [E,e_hidden],
 * "xi" [E,xi_hidden*3], "h" [N,256], "chi" [N,96], "x" [N,3], "fbar" [N,12], "chi_in" [N,6] (state after the
 * last layer).  Writes the shape to rows/cols and, if dst != NULL, copies rows*cols floats to dst (device) on
 * `stream`.  Returns BDIFF_EINVAL for unknown names. */
BDIFF_API int32_t bdiff_debug_tap(bdiff_handle* h, void* stream, const char* which, float* dst, int64_t* rows,
                                  int64_t* cols);

/* Replaces: the arithmetic of EquivariantVariationalDiffusion.sample_p_zs_given_zt
 * (variational_diffusion.py:1204-1278) around the denoiser call:
 *   eps = denoiser(z, t);  mu = z/alpha_ts - c_eps*eps;  z' = mu + sigma*noise;  z'[:, :3] re-centred.
 * noise_x fp32[N,3] and noise_h fp32[N,F] hold the two RAW randn draws of
 * sample_combined_position_feature_noise (:795-819); masking and the centring of noise_x happen inside.
 * z is updated in place.  coef_table: DEVICE array of rows {alpha_ts, c_eps, sigma, t_value} with
 * c_eps = sigma2_ts/alpha_ts/sigma_t and sigma = sigma_ts*sigma_s/sigma_t; the row used is
 * coef_table[*step_index] (step_index: DEVICE int32, or NULL for row 0), so one captured CUDA graph can be
 * replayed for every step while the host only bumps the device counter. */
BDIFF_API int32_t bdiff_reverse_step(bdiff_handle* h, void* stream, float* z, const float* context,
                                     const float* noise_x, const float* noise_h, const float* coef_table,
                                     const int32_t* step_index);

/* Replaces: sample_p_xh_given_z0 up to the normal sample (variational_diffusion.py:840-885):
 *   eps = denoiser(z0, 0);  xh = (1/alpha0)*(z0 - sigma0*eps) + sigma_x*noise (noise masked, x-part centred).
 * coef = {1/alpha0, sigma0, sigma_x, 0} (device).  Writes xh fp32[N,3+F]. */
BDIFF_API int32_t bdiff_decode_z0(bdiff_handle* h, void* stream, const float* z0, const float* context,
                                  const float* noise_x, const float* noise_h, const float* coef, float* xh);

/* Masks two raw randn draws and centres the x-part per molecule (variational_diffusion.py:795-819): z_T. */
BDIFF_API int32_t bdiff_center_noise(bdiff_handle* h, void* stream, const float* noise_x, const float* noise_h,
                                     float* z);

/* Replaces: the RePaint combination inside EquivariantVariationalDiffusion.inpaint (variational_diffusion.py:1659-1667,
 * 1694-1713), run after bdiff_reverse_step has turned z into z_unknown:
 *   z_known = alpha_s*xh0 + sigma_s*noise (compute_noised_representation, :910-931: noise masked, x-part centred over the
 *   molecule);  z_known.x += mean over fixed atoms of (z_unknown.x - z_known.x), per molecule;  z[fixed] = z_known.
 * xh0 fp32[N,3+F] (the input molecule, x centred on its fixed atoms), fixed uint8[N] (1 = atom held fixed), noise_x
 * fp32[N,3] / noise_h fp32[N,F] the two RAW randn draws of the known part.  known_table: DEVICE rows {alpha_s, sigma_s};
 * the row used is known_table[2 * *op_index] (op_index: DEVICE int32), so the call can sit in a replayed CUDA graph.
 * z is updated in place; rows of free atoms and all rows of a molecule without fixed atoms are left unchanged. */
BDIFF_API int32_t bdiff_repaint_combine(bdiff_handle* h, void* stream, float* z, const float* xh0, const uint8_t* fixed,
                                        const float* noise_x, const float* noise_h, const float* known_table,
                                        const int32_t* op_index);

/* Replaces: sample_p_zt_given_zs (variational_diffusion.py:1163-1201; alpha_t|s taken per molecule, i.e. indexed by
 * batch_index where :1177 indexes it by node_mask), the jump back of inpaint (:1730-1749):
 *   z' = alpha_t|s*z + sigma_t|s*noise (noise masked, x-part centred);  z'[:, :3] re-centred.
 * jump_table: DEVICE rows {alpha_t|s, sigma_t|s, s, t}; row jump_table[4 * *jump_index] (DEVICE int32).  In place. */
BDIFF_API int32_t bdiff_renoise(bdiff_handle* h, void* stream, float* z, const float* noise_x, const float* noise_h,
                                const float* jump_table, const int32_t* jump_index);

/* Synchronises `stream` and reports deferred device-side conditions of the work issued so far on this handle.
 * Today: the tile scheduler of the all-layers tensor-core kernel (replaces the kernel boundaries between
 * GCPInteractions layers, gcpnet.py:1161-1176) raises a flag if a dependency wait ever times out; that is an internal
 * error (BDIFF_ECUDA), never expected.  Call after a chain of bdiff_reverse_step / before trusting a result. */
BDIFF_API int32_t bdiff_check(bdiff_handle* h, void* stream);

/* ---- sampling through the C ABI alone ---------------------------------------------------------------------------------
 * Replaces: EquivariantVariationalDiffusion.mol_gen_sample (variational_diffusion.py:1280-1412) as one call, for hosts
 * without torch.  Minimal sequence: bdiff_create -> bdiff_set_weight (every parameter) -> bdiff_prepare ->
 * bdiff_sample_setup -> bdiff_sample (as often as wanted).
 *
 * Noise: counter-based Philox4x32-10 (key = seed, 10 rounds) with Box-Muller, computed inside the step kernels; no
 * generator state.  A chain is a sequence of "draws": buffer fills of N(0, I) values in the order the reference draws
 * them — z_T as draws 0 (x, [N,3]) and 1 (h, [N,F]); reverse step r as draws 2+2r (x) and 3+2r (h); the decode as draws
 * 2+2T and 3+2T.  A chain started from z_init has no z_T draws: everything moves down by 2.  Element e (row-major) of
 * draw d is normal[e & 3] of block (counter = {e >> 2 (64 bit), d (64 bit)}, key = {seed lo, seed hi}): words (w0, w1)
 * give normals 0 and 1, (w2, w3) normals 2 and 3, as r*cos and r*sin of r = sqrt(-2 ln((w_even + 0.5) 2^-32)),
 * angle = 2 pi (w_odd 2^-32), evaluated in double and rounded to float.  The result is a pure function of (seed, d, e).
 * The same seed and batch give bit-identical molecules; the same seed on a different batch composition does not
 * reproduce a molecule (the CoG fix and molecule-boundary effects of the denoiser depend on the whole batch). */

/* The model's sampling constants beyond bdiff_config: num_h must equal num_atom_types + include_charges. */
typedef struct bdiff_sample_config {
  int32_t num_atom_types;    /* A: one-hot columns of h                                                            */
  int32_t include_charges;   /* 0 / 1: h ends with one charge column                                               */
  int32_t model_timesteps;   /* T of the model's gamma table (diffusion_cfg.num_timesteps; 1000 shipped)           */
  int32_t reserved;          /* 0                                                                                  */
  double schedule_power;     /* noise_schedule polynomial_<power> (2 shipped)                                      */
  double noise_precision;    /* diffusion_cfg.noise_precision (1e-5 shipped)                                       */
  float norm_values[3];      /* diffusion_cfg.norm_values: x, one-hot, charges                                     */
  float norm_biases[3];      /* diffusion_cfg.norm_biases; [0] is unused (the reference's None)                    */
} bdiff_sample_config;

/* Host only (no GPU needed): the tables the chain reads, for a chain of num_timesteps steps.  coef_out[num_timesteps*4]
 * receives rows {alpha_ts, c_eps, sigma, t} of reverse steps s = num_timesteps-1 .. 0 (bdiff_reverse_step's table),
 * decode_out[4] = {1/alpha_0, sigma_0, sigma_x, 0} (bdiff_decode_z0's).  gamma is built in fp64 like the reference's
 * PredefinedNoiseSchedule and rounded to fp32 (bit-equal to bdiff/schedule.py's); each coefficient is then evaluated in
 * fp64 from those fp32 gamma values and rounded once, so the tables do not depend on a vector math library or on the
 * CPU.  bdiff/schedule.py evaluates the same formulas in fp32 with torch's CPU kernels, whose result varies with the
 * machine (MKL's exp, SLEEF and the SIMD width torch dispatches to); its c_eps and sigma differ from these by up to
 * ~5e-5 relative at 1000 steps.  To rerun a chain on tables computed elsewhere, pass them to bdiff_sample. */
BDIFF_API int32_t bdiff_schedule_tables(const bdiff_sample_config* cfg, int32_t num_timesteps, float* coef_out,
                                        float* decode_out);

/* Stores the sampling constants on the handle (required before bdiff_sample). */
BDIFF_API int32_t bdiff_sample_setup(bdiff_handle* h, const bdiff_sample_config* cfg);

/* out fp32[rows*cols] (device) <- draw `draw_index` of `seed`: the values the sampling kernels compute internally. */
BDIFF_API int32_t bdiff_noise_fill(void* stream, uint64_t seed, uint64_t draw_index, int64_t rows, int64_t cols,
                                   float* out);
/* out uint32[4*blocks] (device) <- the raw Philox4x32-10 words of blocks 0 .. blocks-1 of draw `draw_index`. */
BDIFF_API int32_t bdiff_philox_fill(void* stream, uint64_t seed, uint64_t draw_index, int64_t blocks, uint32_t* out);

/* The whole chain: z_T (or z_init), num_timesteps reverse steps replayed from one captured CUDA graph (cached on the
 * handle; rebuilt when the batch, the plan or the weights change), the decode, then what mol_gen_sample does last
 * (:1388-1402): argmax one-hot, rounded charges, and the CoG drift fix when the largest per-molecule coordinate sum
 * exceeds 5e-2.  Ends with bdiff_check (synchronises `stream`).
 *   num_nodes_host int32[num_mols] (host) atoms per molecule, all >= 1; no padding mask (every atom is present)
 *   context        fp32[num_mols, num_context] (device), required iff num_context > 0
 *   z_init         fp32[N, 3+num_h] (device, normalised, CoG-free) or NULL; z_init_shape = {N, 3+num_h} (host)
 *   tables_host    NULL (bdiff_schedule_tables) or num_timesteps*4 + 4 floats (host): coef rows then the decode row, to
 *                  run on tables computed elsewhere (bdiff/sampler.py passes its own, so that its chains and this one
 *                  are bit-identical)
 *   xh             fp32[N, 3+num_h] (device) <- [x | one_hot | charges]; batch_index int64[N] (device) or NULL
 * Replans the topology (one D2H + H2D) only when the batch differs from the last call's or another plan intervened. */
BDIFF_API int32_t bdiff_sample(bdiff_handle* h, void* stream, int32_t num_mols, const int32_t* num_nodes_host,
                               const float* context, int32_t num_timesteps, uint64_t seed, const float* z_init,
                               const int64_t* z_init_shape, const float* tables_host, float* xh, int64_t* batch_index);
/* bdiff_sample returning the chain's frames (mol_gen_sample's return_frames, :1309-1310, 1353-1360, 1404-1410):
 * return_frames = F divides num_timesteps; out fp32[F, N, 3+num_h] (device): out[0] = the molecules, without the CoG drift
 * fix (as the reference), out[k] = the unnormalised latent [x * nv0 | h * nv + nb] after the step that lands on
 * s = k * num_timesteps / F.  Same draws as bdiff_sample; bdiff_sample is the case F = 1. */
BDIFF_API int32_t bdiff_sample_frames(bdiff_handle* h, void* stream, int32_t num_mols, const int32_t* num_nodes_host,
                                      const float* context, int32_t num_timesteps, uint64_t seed, const float* z_init,
                                      const int64_t* z_init_shape, int32_t return_frames, const float* tables_host,
                                      float* out, int64_t* batch_index);
/* Number of reverse-step graphs bdiff_sample has captured on this handle (cache diagnostics). */
BDIFF_API int64_t bdiff_sample_graph_builds(const bdiff_handle* h);

/* ---- inpainting through the C ABI alone -------------------------------------------------------------------------------
 * Replaces: EquivariantVariationalDiffusion.inpaint (variational_diffusion.py:1580-1789, RePaint) as one call, with the two
 * repairs of bdiff_renoise / GCDMSampler.inpaint (the dead self-conditioning line is dropped; the jump back takes
 * alpha_t|s per molecule).  Sequence: as for bdiff_sample (bdiff_sample_setup first), then bdiff_inpaint.
 *
 * The RePaint program: get_repaint_schedule (:1549-1578) unrolled into denoise ops (a reverse step to s followed by the
 * combination with the known part) and jumps back from s to s + jump_length.  Draws, in chain order: z_T takes 0 (x) and
 * 1 (h); each op takes 4 (known x, known h, unknown x, unknown h); each jump takes 2 (x, h); the decode takes the last 2.
 * Element layouts and values are those of bdiff_sample's draws, so GCDMSampler.inpaint(noise=philox_noise(seed)) replays
 * the chain.
 *
 * bdiff_repaint_tables (host only): the program for (num_timesteps, num_resamplings, jump_length, return_frames), with
 * the coefficients of bdiff_schedule_tables' precision contract.  *num_ops and *num_jumps are always written; every other
 * output is written when non-NULL, so a call with NULL outputs is the size query:
 *   rev_out   [ops * 4]   {alpha_ts, c_eps, sigma, t} of the op's reverse step (rows of bdiff_schedule_tables)
 *   known_out [ops * 2]   {alpha_s, sigma_s}: z_known = alpha_s * xh0 + sigma_s * noise
 *   jump_out  [jumps * 4] {alpha_t|s, sigma_t|s, s, t}
 *   decode_out[4]         bdiff_schedule_tables' decode row
 *   op_s_out [ops] grid point of the op, slot_out [ops] frame slot (return_frames = no frame), jump_after_out [ops] 0/1,
 *   op_draw_out [ops] / jump_draw_out [jumps] first draw of the op / jump, *decode_draw_out first draw of the decode. */
BDIFF_API int32_t bdiff_repaint_tables(const bdiff_sample_config* cfg, int32_t num_timesteps, int32_t num_resamplings,
                                       int32_t jump_length, int32_t return_frames, int32_t* num_ops, int32_t* num_jumps,
                                       float* rev_out, float* known_out, float* jump_out, float* decode_out,
                                       int32_t* op_s_out, int32_t* slot_out, uint8_t* jump_after_out,
                                       uint64_t* op_draw_out, uint64_t* jump_draw_out, uint64_t* decode_draw_out);

/* The whole inpainting chain: xh0's positions centred on the fixed atoms of each molecule (sequential fp32 sums; a
 * molecule without fixed atoms is not moved), z_T, the RePaint program from two captured CUDA graphs (op and jump, cached
 * on the handle like bdiff_sample's), the decode and bdiff_sample's tail (the CoG drift fix only when return_frames = 1).
 * Ends with bdiff_check (synchronises `stream`).
 *   num_nodes_host, context, batch_index  as in bdiff_sample
 *   xh0_host     fp32[N, 3+num_h] (host) the molecules [x | one_hot | charges], unnormalised as the reference passes them
 *   fixed_host   uint8[N] (host) 1 = the atom keeps its type and position
 *   num_resamplings >= 1, jump_length >= 1; return_frames = F divides num_timesteps and F > 1 needs jump_length = 1
 *   tables_host  NULL (the library's program) or, for a program of O ops and J jumps (bdiff_repaint_tables), O*4 reverse
 *                rows, O*2 known rows, J*4 jump rows and the decode row (host floats) to run on tables computed elsewhere
 *   out          fp32[N, 3+num_h], or [F, N, 3+num_h] with out[0] = the molecules, out[k] = the latent after the op that
 *                lands on s = k * num_timesteps / F (device) */
BDIFF_API int32_t bdiff_inpaint(bdiff_handle* h, void* stream, int32_t num_mols, const int32_t* num_nodes_host,
                                const float* context, int32_t num_timesteps, int32_t num_resamplings, int32_t jump_length,
                                uint64_t seed, const float* xh0_host, const uint8_t* fixed_host, int32_t return_frames,
                                const float* tables_host, float* out, int64_t* batch_index);
/* Number of (op, jump) graph pairs bdiff_inpaint has captured on this handle (cache diagnostics). */
BDIFF_API int64_t bdiff_inpaint_graph_builds(const bdiff_handle* h);

/* ---- optimiser side of a training step (SURVEY.md §8 a21): adaptive gradient-norm clipping + AdamW(amsgrad) + EMA --
 * Replaces, per step: get_grad_norm + Queue statistics + clip_gradients (qm9_mol_gen_ddpm.py:1267-1304,
 * src/models/__init__.py:90-113,442-466), torch.optim.AdamW(lr 1e-4, weight_decay 1e-12, amsgrad) (configs/model/
 * *_mol_gen_ddpm.yaml:3-8) and the EMA callback (src/utils/__init__.py:125-142) by three multi-tensor kernels with
 * no host synchronisation.  All pointers are device pointers owned by the caller.
 *   tensors_dev       one record per parameter tensor (max_exp_avg_sq / ema may be NULL)
 *   chunk_*_dev       the tensors cut into chunks of bdiff_optimizer_chunk() elements: chunk c covers elements
 *                     [chunk_start[c], chunk_start[c] + chunk) of tensor chunk_tensor[c]
 *   partial_dev       scratch, num_chunks doubles
 *   state_dev         BDIFF_OPT_STATE_WORDS 32-bit words, zero-initialised once by the caller and then owned by the
 *                     library: [0] step count (int), [1] history length (int), [2] ring position (int), [3] last
 *                     gradient norm (float), [4] last allowed norm (float), [5] last clip coefficient (float),
 *                     [6] clipped? (int), [8 ...] norm history (floats).  Seed the history like the reference
 *                     (one entry of 3000.0: state[1] = 1, state[2] = 1 % queue_len, state[8] = 3000.0f). */
#define BDIFF_OPT_MAX_QUEUE 120
#define BDIFF_OPT_STATE_WORDS (8 + BDIFF_OPT_MAX_QUEUE)
typedef struct bdiff_opt_tensor {
  float* param;
  const float* grad;
  float* exp_avg;
  float* exp_avg_sq;
  float* max_exp_avg_sq;
  float* ema;
  int64_t numel;
} bdiff_opt_tensor;
typedef struct bdiff_opt_hyper {
  float lr, beta1, beta2, eps, weight_decay, ema_decay;
  int32_t amsgrad;     /* 1: keep the running maximum of exp_avg_sq */
  int32_t clip;        /* 1: clip to 1.5 * mean + 2 * std of the norm history, then push min(norm, limit) */
  int32_t queue_len;   /* history length (reference: 50) */
} bdiff_opt_hyper;
BDIFF_API int32_t bdiff_optimizer_chunk(void);
BDIFF_API int32_t bdiff_optimizer_step(void* stream, const bdiff_opt_tensor* tensors_dev, const int32_t* chunk_tensor_dev,
                                       const int64_t* chunk_start_dev, int32_t num_chunks, double* partial_dev,
                                       int32_t* state_dev, const bdiff_opt_hyper* hyper);

/* ---- post-sampling stability check (SURVEY.md §8 f1) ----------------------------------------------------------------
 * Batched `check_molecular_stability` (src/datamodules/components/edm/__init__.py:91-124 with get_bond_order_batch
 * :61-88): for every molecule k (atoms mol_off[k] .. mol_off[k+1]) the bond order of each atom pair from the three
 * bond-length tables [num_types x num_types] (pm; 0 = no such bond) and margins, the per-atom bond count, and whether
 * that count is allowed for the atom's type (bit c of allowed_mask[type] set <=> c bonds allowed).  Outputs:
 * nr_bonds[N], nr_stable[B] (atoms with an allowed count), mol_stable[B] (1 iff all atoms).  The tables are data of
 * the caller's dataset (the reference keeps them in dataset_info / edm/constants.py); all pointers are device pointers. */
BDIFF_API int32_t bdiff_check_stability(void* stream, const float* x, const int32_t* atom_types, const int32_t* mol_off,
                                        int32_t num_mols, int32_t num_types, const float* bonds1, const float* bonds2,
                                        const float* bonds3, float margin1, float margin2, float margin3,
                                        const uint32_t* allowed_mask, int32_t limit_bonds_to_one, int32_t* nr_bonds,
                                        int32_t* nr_stable, int32_t* mol_stable);

/* Bond-order matrix of `make_mol_edm` (src/datamodules/components/edm/rdkit_functions.py:276-321 with
 * get_bond_order_batch, edm/__init__.py:61-88): for molecule k, bond_order[pair_off[k] + i*n + j] = bond type (0 none, 1, 2, 3)
 * of the pair (i, j) for i > j and 0 otherwise (E = tril(E_full, -1): the directed graph the reference adds to the RWMol),
 * with limit_bonds_to_one = ("GEOM" in dataset_info["name"]).  pair_off int64[B] = exclusive prefix sum of n_k^2.  Same
 * tables / margins as bdiff_check_stability; all pointers are device pointers. */
BDIFF_API int32_t bdiff_bond_orders(void* stream, const float* x, const int32_t* atom_types, const int32_t* mol_off,
                                    const int64_t* pair_off, int32_t num_mols, int32_t num_types, const float* bonds1,
                                    const float* bonds2, const float* bonds3, float margin1, float margin2, float margin3,
                                    int32_t limit_bonds_to_one, int8_t* bond_order);

/* ---- packed training collation (SURVEY.md §8 f3) ---------------------------------------------------------------------
 * Replaces: ProcessedDataset._featurize_as_graph + PyG collation (datamodules/components/edm_dataset.py:187-216: molecules
 * padded to `pad` atoms, mask = charges > 0) and prepare_context (datamodules/components/edm/utils.py:333-382).  The dataset
 * stays on the device in padded form (positions f32[M,pad,3], charges i32[M,pad], one_hot u8[M,pad,A]); a batch = molecule
 * ids idx i64[B].  bdiff_collate_count: counts[k] = present atoms of molecule idx[k].  bdiff_collate_packed: with
 * mol_off i32[B+1] = exclusive prefix sum of the counts, writes the present atoms of the selected molecules in order:
 * x f32[N,3], one_hot f32[N,A], charges f32[N] and batch_index i64[N] — the reference batch restricted to mask == True.
 * bdiff_prepare_context: context[n,c] = (props[c][idx[batch_index[n]]] - mean[c]) / mad[c] for per-molecule properties
 * props f32[C,M] (the reference's global-property branch; the node mask is all ones in a packed batch). */
BDIFF_API int32_t bdiff_collate_count(void* stream, const int32_t* charges, const int64_t* idx, int32_t num_mols, int32_t pad,
                                      int32_t* counts);
BDIFF_API int32_t bdiff_collate_packed(void* stream, const float* positions, const int32_t* charges, const uint8_t* one_hot,
                                       const int64_t* idx, const int32_t* mol_off, int32_t num_mols, int32_t pad,
                                       int32_t num_types, float* x, float* one_hot_out, float* charges_out,
                                       int64_t* batch_index);
BDIFF_API int32_t bdiff_prepare_context(void* stream, const float* props, const int64_t* idx, const int64_t* batch_index,
                                        const float* mean, const float* mad, int64_t dataset_size, int64_t num_nodes,
                                        int32_t num_props, float* context);

/* ---- training pass of the denoiser (SURVEY.md §8 a20) ---------------------------------------------------------------
 * Replaces: loss.backward() through GCPNetDynamics.forward (src/models/components/gcpnet.py:1069-1232) inside
 * EquivariantVariationalDiffusion.forward in .train() mode (variational_diffusion.py:955-1160) — what the Lightning
 * training_step triggers (src/models/qm9_mol_gen_ddpm.py:340-362).
 *
 * Parameters and gradients travel as ONE flat fp32 buffer each, in a canonical layout: the reference tensors (same
 * names and shapes as bdiff_set_weight, nn.Linear weights [out,in] row-major) in ascending name order, each starting at
 * a multiple of 64 floats.  bdiff_param_floats = length of such a buffer; bdiff_param_layout = {offset, count} of one
 * tensor.  A host keeps its nn.Parameters as views of the flat parameter buffer (bdiff/dynamics.py does), so an
 * optimiser step needs no re-upload.
 *
 * bdiff_train_forward: net_out = denoiser(params_flat; xh, t, context) on the current topology plan, same arguments and
 *   result as bdiff_denoise_forward (fp32), and keeps every intermediate the derivative needs (the "tape", device memory
 *   owned by the handle; one tape at a time).
 * bdiff_train_backward: grads_flat <- d/dparams sum(net_out * d_net_out) for the tape of the last bdiff_train_forward
 *   (the buffer is overwritten, not accumulated into).  No atomics: results are bit-reproducible.
 * bdiff_train_precision: tf32 = 0 (default) fp32 GEMMs, 1 = TF32 tensor-core GEMMs (the reference's bf16-mixed training
 *   configuration is the looser of the two).
 * All on `stream`, no host synchronisation.  Errors: BDIFF_ESTATE without a plan / tape, BDIFF_ENOMEM for the tape. */
BDIFF_API int64_t bdiff_param_floats(const bdiff_handle* h);
BDIFF_API int32_t bdiff_param_layout(bdiff_handle* h, const char* name, int64_t* offset, int64_t* count);
BDIFF_API int32_t bdiff_train_precision(bdiff_handle* h, int32_t tf32);
/* Per-operation timing of the training pass: enable = 1 starts recording a CUDA event pair around every kernel and GEMM of
 * the following bdiff_train_forward / bdiff_train_backward calls (on their stream); enable = 0 synchronises `stream`, stops
 * and writes a table (operation, calls, total ms, share; sorted) into report[report_bytes] (NUL-terminated, truncated). */
BDIFF_API int32_t bdiff_train_timing(bdiff_handle* h, void* stream, int32_t enable, char* report, int64_t report_bytes);
BDIFF_API int32_t bdiff_train_forward(bdiff_handle* h, void* stream, const float* params_flat, const float* xh, const float* t,
                                      const float* context, float* net_out);
BDIFF_API int32_t bdiff_train_backward(bdiff_handle* h, void* stream, const float* d_net_out, float* grads_flat);

/* Replaces: the warn-and-zero NaN guard of gcpnet.py:1214-1216 as an observable.  *count_host <- number of denoiser
 * forwards (since the last reset / re-plan of the workspace) in which a NaN position appeared and `vel` was zeroed.
 * Synchronises `stream`.  bench.py reports it for every timed chain. */
BDIFF_API int32_t bdiff_nan_guard_count(bdiff_handle* h, void* stream, int64_t* count_host, int32_t reset);

/* Counters for bench.py: kernels launched by this handle since creation. */
BDIFF_API int64_t bdiff_launch_count(const bdiff_handle* h);

/* ---- EGNN property classifier (inference) -----------------------------------------------------------------------------
 * Replaces: the EDM property classifier the QM9 property-conditional evaluation and the property-optimisation workload
 * score molecules with — EGNN / E_GCL_mask / E_GCL (src/__init__.py:233-419), built by get_classifier (:97-114) and run by
 * test_with_property_classifier (:144-230) on dense batches padded to the largest molecule.  Here molecules are packed
 * (real atoms only): molecule k is atoms mol_off_host[k] .. mol_off_host[k+1] - 1 of x fp32[N,3] and one_hot fp32[N,5],
 * 1 <= n_k <= 128.  bdiff_classifier_forward writes pred fp32[B], the normalised property (EGNN.forward's output); it
 * copies mol_off to the device (the only host work) and never synchronises.  Supported: in_node_nf 5, in_edge_nf 0,
 * hidden_nf 128, either attention and node_attr; anything else -> BDIFF_EINVAL.  set_weight takes the reference's
 * parameter names (embedding.*, gcl_{i}.edge_mlp.{0,2}.*, gcl_{i}.node_mlp.{0,2}.*, gcl_{i}.att_mlp.0.*, node_dec.{0,2}.*,
 * graph_dec.{0,2}.*) as contiguous fp32 device tensors and repacks them on `stream`.  Results are bit-reproducible. */
typedef struct bdiff_classifier bdiff_classifier;
typedef struct bdiff_classifier_config {
  int32_t in_node_nf;   /* 5   */
  int32_t in_edge_nf;   /* 0   */
  int32_t hidden_nf;    /* nf: 128 */
  int32_t n_layers;     /* 1..64 */
  int32_t attention;    /* 0 / 1 */
  int32_t node_attr;    /* 0 / 1 */
} bdiff_classifier_config;
BDIFF_API int32_t bdiff_classifier_create(const bdiff_classifier_config* cfg, bdiff_classifier** out);
BDIFF_API void bdiff_classifier_destroy(bdiff_classifier* h);
BDIFF_API const char* bdiff_classifier_last_error(const bdiff_classifier* h);   /* h may be NULL: last creation error */
BDIFF_API int32_t bdiff_classifier_set_weight(bdiff_classifier* h, void* stream, const char* name, const float* data,
                                              const int64_t* shape, int32_t ndim);
BDIFF_API int32_t bdiff_classifier_forward(bdiff_classifier* h, void* stream, int32_t num_mols, const int32_t* mol_off_host,
                                           const float* x, const float* one_hot, float* pred);

/* ---- training pass of the EGNN property classifier -------------------------------------------------------------------
 * Replaces: loss.backward() through EGNN.forward (src/__init__.py:368-419) in the train branch of
 * train_with_property_classifier (:144-204): the L1 loss of pred against (label - mean) / mad, loss.backward(), then a
 * torch optimiser step.
 *
 * Gradients travel as ONE flat fp32 buffer in a canonical layout: the reference tensors (set_weight's names and shapes,
 * nn.Linear weights [out,in] row-major) in ascending name order, each starting at a multiple of 64 floats.
 * bdiff_classifier_param_floats = length of such a buffer; bdiff_classifier_param_layout = {offset, count} of one tensor.
 *
 * bdiff_classifier_train_forward: same arguments and bit-identical pred as bdiff_classifier_forward, and keeps the tape
 *   (per layer h, the edge_mlp.0 node halves P / Q, agg, node_mlp.0's pre-activation and SiLU; node_dec's and graph_dec's
 *   pre-activations and the molecule sums; copies of x, one_hot and the offsets) in device memory owned by the handle.
 *   One tape per handle: the next training forward replaces it.
 * bdiff_classifier_train_backward: grad_flat <- d/dparams sum_k pred_k d_pred[k] for the tape of the last training
 *   forward (overwritten, not accumulated into; x and one_hot get no gradient).  No atomics: bit-reproducible.
 *   BDIFF_ESTATE without a tape or when set_weight ran after the training forward (the tape's weights are gone).
 * Both on `stream`; the forward copies mol_off to the device, neither synchronises. */
BDIFF_API int64_t bdiff_classifier_param_floats(const bdiff_classifier* h);
BDIFF_API int32_t bdiff_classifier_param_layout(bdiff_classifier* h, const char* name, int64_t* offset, int64_t* count);
BDIFF_API int32_t bdiff_classifier_train_forward(bdiff_classifier* h, void* stream, int32_t num_mols,
                                                 const int32_t* mol_off_host, const float* x, const float* one_hot,
                                                 float* pred);
BDIFF_API int32_t bdiff_classifier_train_backward(bdiff_classifier* h, void* stream, const float* d_pred, float* grad_flat);

#ifdef __cplusplus
}
#endif
#endif /* BDIFF_H_ */
