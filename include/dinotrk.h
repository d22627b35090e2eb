/*
 * dinotrk.h -- C ABI of libdinotrk.so, the H100 (sm_90a) implementation of the
 * DINO-Tracker inference hot path.
 *
 * The reference (AssafSinger94/dino-tracker) has no FFI layer: its boundary is the Python
 * class surface of models/tracker.py + models/model_inference.py (SURVEY.md 8b).  The host
 * mirror of that surface lives in dino_tracker_b200/ and reaches the kernels only through
 * the entry points declared here (ctypes; see INTEGRATION.md).  Every entry point
 *   - is extern "C", takes raw device pointers, sizes and a cudaStream_t (as void*);
 *   - never allocates device memory: big scratch is a caller-provided workspace whose size
 *     comes from the matching *_workspace_bytes query;
 *   - only enqueues work on `stream` unless stated otherwise ("syncs" below);
 *   - returns 0 on success or a negative code; dinotrk_last_error() gives the message
 *     (thread-local).
 *
 * Layouts.  "tpc" = token-major feature video  [T][P][C] fp32, P = h*w tokens row-major
 * (r*w + c), C contiguous: the ViT's natural output order, K-major for every contraction
 * and coalesced for bilinear descriptor sampling.  "chw" = the reference's T x C x h x w
 * (models/tracker.py:64-71).  Pixel coordinates are in the model frame (x in [0,W-1]).
 */
#ifndef DINOTRK_H_
#define DINOTRK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DINOTRK_VERSION 100

#define DINOTRK_OK 0
#define DINOTRK_EINVAL (-22)
#define DINOTRK_ECUDA (-5)
#define DINOTRK_ENOMEM (-12)

/* Video / token-grid geometry.  h = 1 + (H - patch) / stride, w likewise
 * (models/extractor.py:171-177); radius = TrackerHead.argmax_radius (tracker_head.py:47). */
typedef struct dinotrk_geom {
  int H, W, patch, stride, radius;
  int h, w;
} dinotrk_geom;

/* Refiner weights AFTER the spatial-sum normalisation of models/networks/conv_norm.py:34-46
 * (done once per weight load on the host): w1[16][9], b1[16], w2[16][9] (out=1, in=16), b2. */
typedef struct dinotrk_head_weights {
  float w1[16][9];
  float b1[16];
  float w2[16][9];
  float b2;
} dinotrk_head_weights;

/* A cached feature video.  tpc [T][P][C] and norms [T][P] are required.  hi / lo (optional, both or
 * neither): the fp16 split of tpc ([T][P][C] halves each, x = hi + lo) produced by dinotrk_split_fp16; when
 * present the wide correlation groups run on the wgmma tensor cores (3-pass split precision,
 * fp32-faithful), otherwise on the exact-fp32 FFMA GEMM.  C must then be a multiple of 8.
 * q8 / q_fac / q_rho (optional, all or none; C a multiple of 16 and <= 1040): the int8 operands of the anchor phase's
 * coarse pass, written by dinotrk_quantise_s8 with rows_per_group = h*w (q8 [T][P][C] int8, q_fac [T][P], q_rho [T] =
 * the largest relative residual of each frame). */
typedef struct dinotrk_features {
  const float* tpc;
  const float* norms;
  const void* hi;
  const void* lo;
  int T, C;
  const void* q8;
  const float* q_fac;
  const float* q_rho;
} dinotrk_features;

int dinotrk_version(void);
const char* dinotrk_last_error(void);
/* Fills *g from (H, W, patch, stride, radius); returns DINOTRK_EINVAL on bad sizes. */
int dinotrk_make_geom(int H, int W, int patch, int stride, int radius, dinotrk_geom* g);

/* ---- feature cache (models/tracker.py:64-71,131-135) --------------------------------- */
/* chw [T][C][P] -> tpc [T][P][C] and per-token L2 norms [T][P]
 * (frame_embeddings_set.norm(dim=1), models/tracker.py:162). */
int dinotrk_pack_features(const float* chw, float* tpc, float* norms, int T, int C, int P,
                          void* stream);
int dinotrk_unpack_features(const float* tpc, float* chw, int T, int C, int P, void* stream);
int dinotrk_token_norms(const float* tpc, float* norms, int T, int C, int P, void* stream);
/* Per row x of x [rows][C] (fp32 norms [rows], the norms the exact contractions use; C % 16 == 0): s = max|x_k| / 127
 * (fp32), q[row][k] = rint(x_k / s) (int8, [rows][C]), fac[row] = s / max(norm, 1e-4) and the relative residual
 * |x - s q| / |x| (float64, rounded up; 0 for a zero row) into rho[row] (optional) and, as the largest of each group of
 * rows_per_group consecutive rows, into rho_max[ceil(rows / rows_per_group)] (optional). */
int dinotrk_quantise_s8(const float* x, const float* norms, size_t rows, int C, int rows_per_group, void* q, float* fac,
                        float* rho, float* rho_max, void* stream);
/* x = hi + lo with hi = rn_fp16(x), lo = rn_fp16(x - hi) (fp16 arrays of n elements); n % 4 == 0. */
int dinotrk_split_fp16(const float* x, void* hi, void* lo, size_t n, void* stream);
/* The numbers the split's faithful range is stated in: range (device float[2]) = {max |x| over the n elements of x,
 * smallest non-zero value of the n_tok token norms (3.4e38 if there is none)}.  dinotrk_split_faithful (host only) is 1
 * when they are in range for C channels: the split contraction is then fp32-faithful (max |x| <= 65504, every non-zero
 * token norm >= 2^-3 sqrt(C)).  Outside it, give the features without hi / lo: the exact-fp32 GEMM runs instead. */
int dinotrk_split_range(const float* x, size_t n, const float* norms, size_t n_tok, float* range, void* stream);
int dinotrk_split_faithful(float max_abs, float min_norm, int C);

/* ---- descriptor sampling (models/tracker.py:77-111, utils.py:75-101) ------------------- */
/* points [B][3] = (x_px, y_px, set_index) ; frames_set [N] int32 = frame of each set slot.
 * Reproduces normalize_points_for_sampling + the 5-D grid_sample (border, align_corners),
 * including the fp32 temporal-weight leak.  points_normalized != 0: x,y already in [-1,1]
 * (Tracker.sample_embeddings semantics).  out desc [B][C], desc_norm [B] (may be NULL). */
int dinotrk_sample_descriptors(const float* tpc, int T, int C, const dinotrk_geom* g,
                               const float* points, int B, const int* frames_set, int N,
                               int points_normalized, float* desc, float* desc_norm,
                               void* stream);

/* ---- correlation + head (models/tracker.py:158-180, tracker_head.py:107-121) ----------- */
/* Generic grouped form.  Group k (k < n_groups) correlates descriptor rows
 * [row0[k], row0[k] + m[k]) of `desc` with every token of frame frame[k]; its maps are
 * numbered map0[k] + r.  For map j the (x, y) result is written to out[out_index[j] * out_stride
 * + {0,1}] (out_index == NULL: j).  out_mode 0: pixels (after RangeNormalizer.unnormalize,
 * models/model_inference.py:52), 1: normalised [-1,1] (Tracker.forward).
 * group arrays are device int32[n_groups]; total_maps = sum m.  Syncs: no. */
size_t dinotrk_corr_track_workspace_bytes(int total_maps, int n_groups, int C, const dinotrk_geom* g);
int dinotrk_corr_track(const dinotrk_features* feat, const dinotrk_geom* g,
                       const dinotrk_head_weights* hw, const float* desc, const float* desc_norm,
                       const int* grp_frame, const int* grp_row0, const int* grp_m,
                       const int* grp_map0, int n_groups, int total_maps, int max_group_m,
                       const int* out_index, float* out, int out_stride, int out_mode,
                       void* workspace, size_t workspace_bytes, void* stream);

/* Correlation maps only (ReLU'd cosine maps, [total_maps][map_stride] fp32,
 * map_stride = dinotrk_map_stride(g)) -- the volume the fused path never keeps. */
int dinotrk_map_stride(const dinotrk_geom* g);
size_t dinotrk_corr_maps_workspace_bytes(int total_maps, int n_groups, int C);
int dinotrk_corr_maps(const dinotrk_features* feat, const dinotrk_geom* g,
                      const float* desc, const float* desc_norm, const int* grp_frame,
                      const int* grp_row0, const int* grp_m, const int* grp_map0, int n_groups,
                      int total_maps, int max_group_m, float* maps, void* workspace,
                      size_t workspace_bytes, void* stream);
/* Head only: maps -> (x, y) (tracker_head.py:107-121).  aux (may be NULL) receives per map
 * {argmax index, fallback flag} as int32[2].  scratch: device int32[n_maps + 1] enabling the windowed
 * fast path (exact refiner on the 11x11 box around the arg-max + certified absence of the stability
 * branch; uncertified maps go to the full-map kernel); NULL: full-map kernel for every map. */
int dinotrk_head(const float* maps, int n_maps, const dinotrk_geom* g,
                 const dinotrk_head_weights* hw, const int* out_index, float* out,
                 int out_stride, int out_mode, int* aux, int* scratch, void* stream);

/* ---- training: reverse pass of the tracker forward (dino_tracker.py:405-429, models/tracker.py:170-180,303-325) -- */
/* The forward of a training step is dinotrk_sample_descriptors + dinotrk_corr_maps + dinotrk_head (with aux) on the
 * frame set's embeddings, with desc / desc_norm / maps / aux kept.  Given grad_out [B][2] = d loss / d coords (the
 * normalised output of Tracker.forward), row j of points / desc / maps / aux / tgt_frame / grad_out describing map j:
 *   grad_w   float[305] += d loss / d (w1[16][9] | b1[16] | w2[16][9] | b2), w1 / w2 the NORMALISED refiner weights of
 *            dinotrk_head_weights (the spatial-sum normalisation of conv_norm.py:34-46 stays with the caller's autograd);
 *   grad_tpc [T][P][C] += d loss / d feat->tpc, through the target maps (tracker.py:158-169) and through the sampled
 *            source descriptors (tracker.py:96-111); NULL: embeddings without gradient (cached refined features).
 * points [B][3] = (x_px, y_px, set slot) and frames_set [N] as given to dinotrk_sample_descriptors; tgt_frame [B] =
 * the FRAME (index into feat) each map correlates against.  arg-max and disc mask carry no gradient (as in autograd).
 * Accumulates with atomics: the caller zeroes grad_w / grad_tpc.  Syncs: no. */
size_t dinotrk_track_backward_workspace_bytes(int B, int C, const dinotrk_geom* g);
int dinotrk_track_backward(const dinotrk_features* feat, const dinotrk_geom* g, const dinotrk_head_weights* hw,
                           const float* points, const int* frames_set, int N, const float* desc,
                           const float* desc_norm, const int* tgt_frame, const float* maps, const int* aux,
                           const float* grad_out, int B, float* grad_w, float* grad_tpc, void* workspace,
                           size_t workspace_bytes, void* stream);

/* Reverse pass of dinotrk_sample_descriptors alone (the contrastive losses sample refined embeddings with a graph,
 * dino_tracker.py:215-220): grad_tpc [T][P][C] += the trilinear weights of every point times grad_desc [B][C]. */
int dinotrk_sample_backward(int T, int C, const dinotrk_geom* g, const float* points, int B, const int* frames_set,
                            int N, int points_normalized, const float* grad_desc, float* grad_tpc, void* stream);

/* ---- inference driver (models/model_inference.py:97-216) ------------------------------- */
/* query_points [N][3] (x, y, t) px; frame_batch = the reference's --batch-size (0 = whole
 * video).  Outputs: traj [N][T][3] (x, y, t); cos_sims [N][T]; anchors [N][T(a)][T(i)][2] valid
 * where cos_sims[n][a] >= anchor_th; occ [N][T] uint8.  Any of the last three may be NULL only
 * together with stop_after < 3 / 2 / 1.  Phases 0 = trajectories (compute_trajectories),
 * 1 = cos-sims, 2 = anchors, 3 = occlusion; phases start_phase..stop_after run (0..3 = infer), and
 * the outputs of earlier phases are then inputs.  SYNCS the stream once when phase 2 runs (reads
 * the per-frame anchor counts back to size the anchor work lists). */
size_t dinotrk_infer_workspace_bytes(int T, int C, const dinotrk_geom* g, int N, int chunk_maps);
/* Host-only helper (no GPU needed): the chunk plan dinotrk_infer uses.  kind 0 = trajectory phase (items = every
 * (frame, query row) pair), kind 1 = anchor phase (anchor_counts[a] * T items per anchor frame a).  Chunks hold
 * <= chunk_maps correlation maps; inside a chunk the items of one target frame form a group.  Outputs (either may be
 * NULL to just count): groups [n_chunks][5][T + 2] int32 = per chunk {frame, first descriptor row, rows m, first map,
 * first item} x group; meta [n_chunks][4] = {maps used, largest m, number of groups, 1 if no group is thin};
 * *n_chunks.  dinotrk_infer_max_chunks bounds n_chunks (and sizes dinotrk_infer's workspace). */
size_t dinotrk_infer_max_chunks(int T, int N, int chunk_maps);
int dinotrk_infer_plan(int kind, int T, int N, const int* anchor_counts, int chunk_maps, int* groups, int* meta,
                       int max_chunks, int* n_chunks);
/* Host-only helper: the anchor-phase plan of pipeline 1 (coarse pass + exact window), which reads descriptor rows in place
 * where it can.  Descriptor rows are numbered in one space: row n T + i (< N T) is the unique sample of trajectory point i
 * of query n; the rows behind belong to a ring of 4 chunks, map j of chunk k at N T + (k % 4) ch + j with
 * ch = max(chunk_maps, T).  qlist [T][N]: the queries anchored at frame a, ascending, anchor_counts[a] of them;
 * query_flag [N]: 1 = the query's descriptors depend on the anchor frame, it is never read in place.  Chunks are cut at
 * whole (query, anchor frame) cells of T items (probe != 0: a first chunk of <= 4096 maps); a frame's span of a chunk is
 * cut into groups at its runs of consecutive unflagged queries.  A run is read in place (first row = first query * T) when
 * padding it to 256-row tiles costs at most 1/16 of its rows; the other cells are gathered (first row = the chunk's row of
 * the group's first map), adjacent ones as one group.  groups [n_chunks][5][gcap] as above with
 * gcap = dinotrk_infer_anchor_gcap(T, chunk_maps); meta [n_chunks][5] = {maps used, largest m, number of groups, 1 if no
 * group is thin, gathered maps}.  Either may be NULL to just count. */
int dinotrk_infer_anchor_gcap(int T, int chunk_maps);
int dinotrk_infer_plan_anchors(int T, int N, const int* anchor_counts, const int* qlist, const unsigned char* query_flag,
                               int chunk_maps, int probe, int* groups, int* meta, int max_chunks, int* n_chunks);
/* Phase 2 pipelining across CUDA streams (process-wide; results are identical in every mode):
 * 0 = everything on the caller's stream; 1 (default) = the descriptor sampling of chunk k+1 runs on an
 * internal side stream under the correlation GEMM of chunk k; 2 = the head's fast path as well;
 * -1 = back to the default / the DTK_OVERLAP environment variable.  All side-stream work is joined back
 * into the caller's stream before dinotrk_infer returns.  The side streams and their events are one set per
 * process (one process per GPU): with mode >= 1 do not run dinotrk_infer from two host threads at once. */
int dinotrk_infer_set_overlap(int mode);
/* Pipeline of the anchor re-tracking phase (process-wide):
 *  1 = coarse pass + exact window: one single-pass fp16 GEMM keeps per map and 128-token tile only (max, its token, second
 *      value); the fp32-faithful split-precision contraction is then evaluated only on a 21 x 21 token box around the
 *      arg-max of each (query, anchor frame) cell, and a warp-per-map head consumes those values -- no correlation map is
 *      ever written.  Maps whose arg-max cannot be resolved from the coarse pass (near ties), that leave their cell's box
 *      or that fail the head's certificate are re-done by pipeline 0; no result depends on a coarse value.
 *  0 = full maps: split-precision GEMM over all tokens into chunk buffers + the head kernels (the round-1 pipeline).
 * -1 (default) = 1 when the feature struct carries fp16 hi / lo halves (tensor path), unless the trajectory phase just
 *      showed that the head's certificate fails for more than a quarter of the maps (ill-conditioned refiner weights);
 *      the DTK_XW environment variable (0 / 1) overrides.
 * dinotrk_infer_last_stats (n >= 4 slots): {anchor-phase maps, maps finished by the exact-window path, maps re-done by the
 * full-map path, pipeline used[, of the re-done maps: those queued by the head's certificate rather than by the plan[,
 * contraction: 1 = split fp16 tensor cores, 0 = exact fp32[, coarse pass of pipeline 1: 1 = int8, 0 = fp16 (the pass the
 * phase finished with)[, bits of the float max over frames of feat->q_rho, 0 without int8 operands[, maps of pipeline 1
 * whose descriptor the GEMMs read in place from the unique (query, source frame) table, maps whose descriptor was gathered
 * into the chunk's rows]]]]]} of the last dinotrk_infer call that ran the anchor phase. */
int dinotrk_infer_set_path(int path);
/* Coarse pass of pipeline 1:  1 = int8 (feat->q8 required),  0 = fp16 over feat->hi,
 * -1 (default) = int8 when feat->q8 is given and every frame's q_rho is <= 0.03, unless the probe chunk queues more than
 *      1/16 of its maps to pipeline 0; fp16 otherwise.  No result depends on the choice. */
int dinotrk_infer_set_coarse(int mode);
int dinotrk_infer_last_stats(long long* out, int n);
/* The coarse pass of pipeline 1 on its own (for testing its keys): the single-pass fp16 GEMM of desc_hi [desc_rows][C]
 * (fp16, the `hi` half of the descriptors) against feat->hi, group k correlating rows [grp_row0[k], grp_row0[k] + grp_m[k])
 * with frame grp_frame[k] (device int32[n_groups]).  For descriptor row j and 128-token tile t (n_tiles = ceil(h*w / 128)):
 * key1[j][t] = bits(max) << 32 | (0x7fffffff - first token holding it) and max2[j][t] = the second largest value of the
 * tile, both of relu(coarse dot / max(|d| |F|)) with |d| = desc_norm[j], |F| = feat->norms (clamped at 1e-4).  Rows
 * outside every group are not written.  feat->hi is required. */
size_t dinotrk_xw_coarse_keys_workspace_bytes(int T, int n_groups, const dinotrk_geom* g);
int dinotrk_xw_coarse_keys(const dinotrk_features* feat, const dinotrk_geom* g, const void* desc_hi, int desc_rows,
                           const float* desc_norm, const int* grp_frame, const int* grp_row0, const int* grp_m, int n_groups,
                           unsigned long long* key1, float* max2, void* workspace, size_t workspace_bytes, void* stream);
/* The same keys from the int8 pass: values relu(<desc_q8[j], feat->q8[frame][p]> desc_fac[j] feat->q_fac[frame][p])
 * (desc_q8 int8 [desc_rows][C], desc_fac [desc_rows], desc_rho [desc_rows]: dinotrk_quantise_s8 of the descriptors).
 * eps[j] (optional, float [desc_rows], rows of the groups only) receives the per-map bound on |coarse - exact cosine| the
 * plan uses, from desc_rho[j] and feat->q_rho[frame].  feat->q8, q_fac and q_rho are required.  Workspace: as above. */
int dinotrk_xw_coarse_keys_i8(const dinotrk_features* feat, const dinotrk_geom* g, const void* desc_q8, const float* desc_fac,
                              const float* desc_rho, int desc_rows, const int* grp_frame, const int* grp_row0, const int* grp_m,
                              int n_groups, unsigned long long* key1, float* max2, float* eps, void* workspace,
                              size_t workspace_bytes, void* stream);
/* The exact box GEMM of pipeline 1 on its own (for testing and timing it): per cell k (device int32[n_cells] arrays), the
 * split-precision contraction (lo*hi + hi*lo + hi*hi, the full-map GEMM's sequence) of descriptor rows
 * [cell_row0[k], cell_row0[k] + cell_m[k]) (desc_hi / desc_lo: fp16 [desc_rows][C], dinotrk_split_fp16 of the fp32 rows)
 * against the 21 x 21 token box of frame cell_frame[k] whose first row / column is box_org[k] = {row, column} (int32
 * [n_cells][2]; tokens outside the grid count as zero; column INT_MIN: skip the cell).  Writes the raw accumulators
 * xbox[row][by * 21 + bx] (fp32, [desc_rows][448]); columns 441..447, rows outside every cell and the rows of skipped cells
 * are not written.  max_m = the largest cell_m (<= 128).  feat->hi and feat->lo are required.  Syncs: no. */
int dinotrk_xw_box_gemm(const dinotrk_features* feat, const dinotrk_geom* g, const void* desc_hi, const void* desc_lo,
                        int desc_rows, const int* cell_row0, const int* cell_m, const int* cell_frame, const int* box_org,
                        int n_cells, int max_m, float* xbox, void* stream);
int dinotrk_infer(const dinotrk_features* feat, const dinotrk_geom* g,
                  const dinotrk_head_weights* hw, const float* query_points, int N,
                  float anchor_th, float cos_th, int frame_batch, int start_phase, int stop_after,
                  int chunk_maps,
                  float* traj, float* cos_sims, float* anchors, uint8_t* occ,
                  void* workspace, size_t workspace_bytes, void* stream);
/* Piecewise entry points behind ModelInference.compute_* (same arithmetic as dinotrk_infer). */
int dinotrk_traj_cos_sims(const float* tpc, int T, int C, const dinotrk_geom* g,
                          const float* traj, const float* query_points, int N, float* cos_sims,
                          void* workspace, size_t workspace_bytes, void* stream);
int dinotrk_occlusion(const float* traj, const float* cos_sims, const float* anchors, int N, int T,
                      float anchor_th, float cos_th, uint8_t* occ, void* stream);

/* ---- Delta-DINO refinement (models/tracker.py:113-135, delta_dino.py:8-61, models/utils.py:7-45) */
/* frames [B][3][H][W] raw RGB in [0,1]; channels[5] = {3, c1, c2, c3, C} (c* multiples of 4);
 * wgt[l] = conv l weights with BatchNorm(eval) folded in, K-major [C_out][5][5][C_in_pad]
 * (C_in_pad = 4 for l = 0, else C_in); bias[l] [C_out] likewise folded.  dino_tpc [B][h*w][C];
 * ixs[w] / iys[h] = un-normalised clipped CNN-grid sampling coordinates of the token columns / rows
 * (models/utils.py:31-43).  Writes refined_tpc [B][h*w][C] = dino + aligned residual and
 * (optional) per-token norms [B][h*w]. */
size_t dinotrk_delta_workspace_bytes(int B, int H, int W, const int* channels);
int dinotrk_delta_refine(const float* frames, int B, int H, int W, const int* channels,
                         const float* const* wgt, const float* const* bias, const float* dino_tpc,
                         const float* ixs, const float* iys, int h, int w, float* refined_tpc,
                         float* norms, void* workspace, size_t workspace_bytes, void* stream);

/* Frame-sharded multi-GPU variant (SURVEY.md 8e, config 4): as dinotrk_delta_refine, and every refined row is ALSO
 * stored into the same slot of each peer GPU's full feature video -- peer_bases[k] (HOST array of n_peers <= 8 device
 * pointers mapped with dinotrk_peer_open) + (first_frame * h*w + row) * C -- by the producing kernel itself
 * (stores over NVLink to mapped peer memory): the all-gather is fused into the delta-DINO epilogue.  The caller
 * synchronises the ranks afterwards (stream sync + barrier) before reading remote frames. */
int dinotrk_delta_refine_allgather(const float* frames, int B, int H, int W, const int* channels,
                                   const float* const* wgt, const float* const* bias, const float* dino_tpc,
                                   const float* ixs, const float* iys, int h, int w, float* refined_tpc,
                                   float* norms, void* workspace, size_t workspace_bytes,
                                   float* const* peer_bases, int n_peers, size_t first_frame, void* stream);
/* Tensor-core variant: the four convolutions run as explicit-im2col (fp16 hi/lo split on the fly) + wgmma
 * split-precision GEMMs (fp32-faithful).  wgt_hi[l] / wgt_lo[l]: fp16 split (dinotrk_split_fp16) of the folded K-major
 * weights [C_out][Kp], Kp = 25 * C_in_pad rounded up to 8; channel counts multiples of 8.  peer_bases / n_peers /
 * first_frame as in dinotrk_delta_refine_allgather (n_peers = 0: single GPU). */
int dinotrk_delta_refine_tc(const float* frames, int B, int H, int W, const int* channels,
                            const void* const* wgt_hi, const void* const* wgt_lo, const float* const* bias,
                            const float* dino_tpc, const float* ixs, const float* iys, int h, int w,
                            float* refined_tpc, float* norms, void* workspace, size_t workspace_bytes,
                            float* const* peer_bases, int n_peers, size_t first_frame, void* stream);
/* Peer-mapped buffers for the above (one process per GPU, one node): cudaMalloc + CUDA IPC handle (64 bytes). */
int dinotrk_peer_alloc(size_t bytes, void** ptr, unsigned char* handle64);
int dinotrk_peer_open(const unsigned char* handle64, void** ptr);
int dinotrk_peer_close(void* ptr);
int dinotrk_peer_free(void* ptr);

/* ---- Delta-DINO training step (delta_dino.py:22-61 with gradients, models/tracker.py:113-129) -------------------
 * One chunk of B frames (the reference's 8-frame batches; each chunk is its own BatchNorm batch).  channels[5] =
 * {3, c1, c2, c3, C}, c* multiples of 8; every reflect pad must be smaller than the map it pads (as torch requires).
 * Forward: wgt_hi[l] / wgt_lo[l] = fp16 split (dinotrk_split_fp16) of the UNFOLDED conv weights, K-major
 * [C_out][5][5][C_in_pad] with K padded to Kp = 25 * C_in_pad rounded up to 8 (C_in_pad = 4 for l = 0); conv_bias,
 * bn_weight (gamma), bn_bias (beta), running_mean, running_var: [C_out] per layer.  training = 1: BatchNorm on the
 * batch statistics (float64 two-pass reduction over B*H*W) and the running statistics updated in place as
 * torch.nn.BatchNorm2d does (momentum, unbiased running_var; num_batches_tracked is the caller's); training = 0: the
 * running statistics, left unchanged.  Writes residual_tpc [B][h*w][C] = the aligned BN output of the last layer
 * (ixs / iys as in dinotrk_delta_refine) and fills `saved` (dinotrk_delta_train_saved_bytes: the pre-BN conv outputs and
 * the per-channel statistics) for the backward.  B = 0 writes nothing.  Syncs: no.
 * Backward: grad_residual_tpc [B][h*w][C]; wgtT_hi[l] / wgtT_lo[l] (l = 1..3, entry 0 unused) = fp16 split of the conv
 * weights transposed to [C_in][5][5][C_out]; bn_weight / bn_bias / training and `saved` as given to the forward.  WRITES
 * (does not accumulate) grad_wgt[l] [C_out][Kp] in the forward's K-major layout (columns past 25 * C_in_pad are zero),
 * grad_bias[l], grad_bn_weight[l], grad_bn_bias[l] [C_out].  Frames get no gradient.  Every reduction runs in a fixed
 * order: results are bit-for-bit reproducible.  The convolution GEMMs run on fp16 hi / lo splits; each gradient operand
 * is scaled by a power of two from its max |.| first (exact), so the result does not depend on the gradient's scale.
 * Syncs: no. */
size_t dinotrk_delta_train_saved_bytes(int B, int H, int W, const int* channels);
size_t dinotrk_delta_train_forward_workspace_bytes(int B, int H, int W, const int* channels);
size_t dinotrk_delta_train_backward_workspace_bytes(int B, int H, int W, const int* channels);
int dinotrk_delta_train_forward(const float* frames, int B, int H, int W, const int* channels, const void* const* wgt_hi,
                                const void* const* wgt_lo, const float* const* conv_bias, const float* const* bn_weight,
                                const float* const* bn_bias, float* const* running_mean, float* const* running_var,
                                int training, float momentum, float eps, const float* ixs, const float* iys, int h, int w,
                                float* residual_tpc, void* saved, size_t saved_bytes, void* workspace, size_t workspace_bytes,
                                void* stream);
int dinotrk_delta_train_backward(const float* frames, int B, int H, int W, const int* channels, const void* const* wgtT_hi,
                                 const void* const* wgtT_lo, const float* const* bn_weight, const float* const* bn_bias,
                                 int training, const float* ixs, const float* iys, int h, int w, const float* grad_residual_tpc,
                                 const void* saved, size_t saved_bytes, float* const* grad_wgt, float* const* grad_bias,
                                 float* const* grad_bn_weight, float* const* grad_bn_bias, void* workspace,
                                 size_t workspace_bytes, void* stream);

/* ---- DINOv2 ViT feature extractor (utils.py:32-72, models/extractor.py:41-85,137-150) -------------- */
typedef struct dinotrk_vit_config {
  int depth, dim, heads;   /* ViT-L/14: 24, 1024, 16; ViT-B/14: 12, 768, 12 (head dim 64) */
  int tap_layer;           /* 0-based block whose output (before the final norm) is returned; 15 in the shipped config */
  int patch, stride;       /* 14, 7 */
  int attn_materialized;   /* 0: fused wgmma attention (fp16 q/k/v/p, scores stay on the SM); 1: TF32 scores through a
                              workspace (tensor-core GEMM -> softmax -> tensor-core GEMM), validation path */
  int gemm_f16;            /* 1: linear layers on the fp16 tensor pipe -- patch_w and the qkv / proj / fc1 / fc2 weight matrices
                              are passed as fp16 arrays, activations are written in fp16 by the producing epilogue;
                              0 (or attn_materialized): fp32 arrays, TF32 MMAs */
  int gemm_pair;           /* with gemm_f16: 1 = linear layers on CTA pairs (two-CTA clusters, 256 x 256 tiles, each CTA
                              loads half of the weight tile and multicasts it to both), 0 = single-CTA 128 x 256 tiles */
} dinotrk_vit_config;
/* Device fp32 (weight matrices fp16 when gemm_f16).  patch_w: patch-embedding conv weight flattened K-major
 * [dim][Kp], Kp = 3*patch*patch zero-padded to a multiple of 4 (fp32) / 8 (fp16) elements; cls_pos [dim] =
 * cls_token + pos_embed[0]; pos [h*w][dim] = bicubic-interpolated patch position embedding (extractor.py:57-85);
 * blocks: HOST array of depth x 14 device pointers in the order norm1.w, norm1.b, qkv.w [3D][D], qkv.b, proj.w,
 * proj.b, ls1.gamma, norm2.w, norm2.b, fc1.w [4D][D], fc1.b, fc2.w [D][4D], fc2.b, ls2.gamma. */
typedef struct dinotrk_vit_weights {
  const void* patch_w; const float* patch_b; const float* cls_pos; const float* pos;
  const float* const* blocks;
} dinotrk_vit_weights;
size_t dinotrk_vit_workspace_bytes(const dinotrk_vit_config* c, const dinotrk_geom* g, int B);
/* frames [B][3][H][W] RGB in [0,1] -> out_tpc [B][h*w][dim] (token-major features of block tap_layer). */
int dinotrk_vit_forward(const float* frames, int B, const dinotrk_geom* g, const dinotrk_vit_config* c,
                        const dinotrk_vit_weights* wt, float* out_tpc, void* workspace,
                        size_t workspace_bytes, void* stream);
/* The attention of one ViT block on its own (the fused wgmma kernel of dinotrk_vit_forward; head dim 64):
 * q16 [B*heads][N1][64] fp16 ALREADY multiplied by 64^-1/2 * log2(e), k16 [B*heads][N1][64] fp16,
 * vT16 [B*heads][64][N1p] fp16 (v transposed, row pitch N1p >= N1, a multiple of 8);
 * out [B*N1][heads*64] fp32 = softmax(q k^T) v with head h in columns [64 h, 64 h + 64)
 * (the layout of the reference's attn output before `proj`, dinov2 attention.py). */
int dinotrk_vit_attention(const void* q16, const void* k16, const void* vT16, int B, int heads, int N1, int N1p,
                          float* out, void* stream);
/* The same with an fp16 out16 [B*N1][heads*64]: the store the forward's fp16 operand mode feeds to `proj`. */
int dinotrk_vit_attention_f16(const void* q16, const void* k16, const void* vT16, int B, int heads, int N1, int N1p,
                              void* out16, void* stream);
/* One stage of dinotrk_vit_forward on its own, with the forward's own code, for testing and timing the layers
 * (fp16 operand mode: c->gemm_f16 = 1, c->attn_materialized = 0; c->gemm_pair picks CTA pairs or single CTAs for
 * qkv / proj / fc1 / fc2).  N1 = g->h * g->w + 1 tokens per frame, rows = B * N1, D = c->dim, fp16 weight matrices
 * K-major as in dinotrk_vit_weights, fp32 parameter vectors.  Per stage (in, w, p0, p1 -> out0 [, out1, out2]):
 *   LAYERNORM  x [rows][D] fp32, -, weight [D], bias [D]  -> y [rows][D] fp16   (eps 1e-6)
 *   PATCH      cols [B*h*w][Kp] fp16 (Kp = 3*patch*patch rounded up to 8), patch_w [D][Kp], bias [D], pos [h*w][D]
 *              -> x [B][N1][D] fp32: x[b][1 + p] = cols[b*h*w + p] . patch_w + bias + pos[p]; x[b][0] is not written
 *   QKV        y [rows][D] fp16, qkv_w [3D][D], bias [3D], -  -> q [B*heads][N1][64] fp16 multiplied by
 *              64^-1/2 * log2(e), k [B*heads][N1][64] fp16, vT [B*heads][64][N1p8] fp16 (v transposed, row pitch N1p8 =
 *              N1 rounded up to 8; columns N1..N1p8-1 are not written): dinotrk_vit_attention's inputs
 *   PROJ       y [rows][D] fp16, proj_w [D][D], bias [D], ls [D]  -> x [rows][D] fp32 += ls * (y . proj_w + bias)
 *   FC1        y [rows][D] fp16, fc1_w [4D][D], bias [4D], -  -> h [rows][4D] fp16 = gelu(y . fc1_w + bias) (exact GELU
 *              with erf to 1.5e-7)
 *   FC2        h [rows][4D] fp16, fc2_w [D][4D], bias [D], ls [D]  -> x [rows][D] fp32 += ls * (h . fc2_w + bias)
 * workspace: DINOTRK_VIT_STAGE_WORKSPACE_BYTES of device memory (tile plan).  Rows past `rows` are not touched. */
#define DINOTRK_VIT_LAYERNORM 0
#define DINOTRK_VIT_PATCH 1
#define DINOTRK_VIT_QKV 2
#define DINOTRK_VIT_PROJ 3
#define DINOTRK_VIT_FC1 4
#define DINOTRK_VIT_FC2 5
#define DINOTRK_VIT_STAGE_WORKSPACE_BYTES 4096
int dinotrk_vit_stage(int stage, const dinotrk_vit_config* c, const dinotrk_geom* g, int B, const void* in, const void* w,
                      const float* p0, const float* p1, void* out0, void* out1, void* out2, void* workspace,
                      size_t workspace_bytes, void* stream);

/* ---- best buddies (preprocessing_dino_bb/extract_dino_best_buddies.py:12-54) ------------------------ */
/* For every ordered pair k (source frame pair_src[k], target frame pair_tgt[k]; device int32[n_pairs]):
 * nn_idx[k][n] = argmax_m cos(F_src[n], F_tgt[m]) (first maximum), nn_cos[k][n] = that cosine (exact fp32,
 * clamp 1e-8 on the norm product).  The affinity matrix runs through the wgmma split-fp16 GEMM and never
 * leaves the SM; candidates are re-evaluated in exact fp32.  feat->hi / lo are required. */
size_t dinotrk_best_buddies_workspace_bytes(int n_pairs, int P);
int dinotrk_best_buddies_pairs(const dinotrk_features* feat, const dinotrk_geom* g, const int* pair_src,
                               const int* pair_tgt, int n_pairs, int* nn_idx, float* nn_cos,
                               void* workspace, size_t workspace_bytes, void* stream);
/* mutual[k][n] = (nn_ts[k][nn_st[k][n]] == n): source token n of pair k is a best buddy. */
int dinotrk_bb_mutual(const int* nn_st, const int* nn_ts, int n_pairs, int P, uint8_t* mutual, void* stream);
/* Peak filter of the best-buddy pairs (preprocessing_dino_bb/compute_dino_bb_nms.py:12-66, get_bb_sim_indices): maps =
 * [n_maps][dinotrk_map_stride] similarity maps of the source points against the target frame (dinotrk_corr_maps). Per map:
 * peak_affs[2] = the two largest values that survive box NMS (boxes of +-box_size px around the token centres, greedy,
 * IoU threshold, restricted to the `topk` largest values), r = second / first. */
int dinotrk_bb_nms(const float* maps, int n_maps, const dinotrk_geom* g, float box_size, float iou_thresh, int topk,
                   float* peak_affs, float* r, void* stream);

/* ---- optical-flow trajectories (preprocessing/extract_trajectories.py) ------------------------------------------ */
/* The flows of a T-frame H x W video: fwd[i] / bwd[i] = flow from frame i to i+1 / from i+1 to i, [T-1][2][H][W]
 * fp32 (channel 0 = x).  Flows are sampled as data/data_utils.py bilinear_sampler does (grid_sample, zeros padding,
 * align_corners), norms are fp32 sqrt(dx*dx + dy*dy). */
typedef struct dinotrk_flow_video {
  const float* fwd;
  const float* bwd;
  int T, H, W;
} dinotrk_flow_video;
/* get_flows_with_masks (extract_trajectories.py:61-95): masks [T+1][H][W] uint8; masks[i+1] = 1 where the round trip
 * frame i+1 -> i -> i+1 returns within `threshold` px AND some pixel of frame i warps (rounded) onto the pixel.
 * masks[0] = masks[T] = 0. */
int dinotrk_flow_masks(const dinotrk_flow_video* fv, float threshold, uint8_t* masks, void* stream);
/* Chaining of one start frame s (extract_trajectories.py:203-266).  dinotrk_traj_chain walks every pixel of frame s
 * that starts a trajectory (masks[s] == 0, or no trajectory kept from an earlier start frame passes through it) through
 * frames s+1.. while the cycle check (< threshold), the bounds check and, when direct flows are given, the direct-flow
 * check (< direct_threshold, :98-160 and :222-255) hold; direct_fwd / direct_bwd = [T-1-s][2][H][W] flows s -> s+1+k /
 * s+1+k -> s.  It writes the number of trajectories of at least min_len frames to *n_kept (device int).
 * dinotrk_traj_emit then writes them to out [n_kept][T][2] (NaN outside their frames), in row-major pixel order, and
 * records their rounded positions for the look-behind of later start frames.  Run s = 0, 1, ... in order, chain then
 * emit, on one workspace zeroed before s = 0. */
size_t dinotrk_traj_workspace_bytes(int T, int H, int W);
int dinotrk_traj_chain(const dinotrk_flow_video* fv, const uint8_t* masks, int s, float threshold, int min_len,
                       const float* direct_fwd, const float* direct_bwd, float direct_threshold, int* n_kept,
                       void* workspace, size_t workspace_bytes, void* stream);
int dinotrk_traj_emit(const dinotrk_flow_video* fv, int s, float* out, void* workspace, size_t workspace_bytes, void* stream);

/* ---- optical-flow filter of the best buddies (preprocessing_dino_bb/of_filter_dino_best_buddies.py) ------------- */
/* nearest [T][gh][gw] int32 = argmin_n |traj[n][t] - g| over trajectories traj [M][T][2] for the grid points
 * g = (start + step j, start + step i) (create_meshgrid); a NaN position is never nearest, ties -> lowest n, a frame
 * without any valid position -> 0 (torch.argmin over +inf).  Exact: distances are fp32 sqrt(dx*dx + dy*dy). */
size_t dinotrk_traj_nearest_workspace_bytes(int M, int T, int gh, int gw);
int dinotrk_traj_nearest(const float* traj, int M, int T, int gh, int gw, float start, float step, int* nearest,
                         void* workspace, size_t workspace_bytes, void* stream);
/* The pair filter (:86-97) over all ordered pairs at once.  Pair k (frames pair_src[k] -> pair_tgt[k]) owns points
 * [offsets[k], offsets[k+1]) of src_xy / tgt_xy [n_pts][2] (pixel coordinates).  keep[i] = 1 when the nearest
 * trajectory of the source point's grid cell ((p - 7) // stride) is NaN at the target frame AND that of the target point
 * is NaN at the source frame: the pairs the flow does not cover. */
int dinotrk_of_filter(const float* traj, int M, int T, const int* nearest, int gh, int gw, int stride, const float* src_xy,
                      const float* tgt_xy, const int* pair_src, const int* pair_tgt, const int* offsets, int n_pairs, int n_pts,
                      uint8_t* keep, void* stream);

/* ---- foreground masks (preprocessing/create_fg_mask.py) and the fg / bg split (split_trajectories_to_fg_bg.py) ---- */
/* The features are token-major fp32 rows a [M][C] (M = T*h*w, the ViT's output), C % 4 == 0, C <= 1536, 16-byte
 * aligned; q <= 4.  Offsets are 64-bit.  Every sum runs in a fixed order: two runs give the same bits.
 * dinotrk_pca_stats: s [M] = 1 / max(|a_i|, 1e-12) (F.normalize's rule; 1 when normalize == 0) and c [C] = the column
 * mean of diag(s) A (float64 partials over fixed row ranges).
 * dinotrk_pca_power: one read of the rows gives X = (diag(s) A - 1cᵀ) P [M][q] and W = (diag(s) A - 1cᵀ)ᵀ X [C][q] for
 * P [C][q]: with QR(X) = Q R, the next iterate of torch.pca_lowrank's subspace iteration is W R⁻¹.
 * Both take a workspace of dinotrk_pca_workspace_bytes(M, C, q) bytes (q = 1 for the stats). */
size_t dinotrk_pca_workspace_bytes(long long M, int C, int q);
int dinotrk_pca_stats(const float* a, long long M, int C, int normalize, float* s, float* c, void* workspace,
                      size_t workspace_bytes, void* stream);
int dinotrk_pca_power(const float* a, long long M, int C, int q, const float* s, const float* c, const float* P, float* X,
                      float* W, void* workspace, size_t workspace_bytes, void* stream);
/* create_fg_mask.py:29-42: colors [M][q] = diag(s) A V (not centred), token_mask [T][h][w] = 1 where
 * (colors[:,0] - min) / (max - min) < threshold (fp32), and mask [T][H][W] = 255 * its nearest upsampling.  workspace:
 * 32 bytes. */
int dinotrk_fg_mask(const float* a, int T, int h, int w, int C, int q, const float* s, const float* V, float threshold,
                    int H, int W, float* colors, uint8_t* token_mask, uint8_t* mask, void* workspace, size_t workspace_bytes,
                    void* stream);
/* F.interpolate(mode="nearest") of a 0/1 token mask [T][h][w] to [T][H][W] 0/255: source index
 * min((int)floorf(dst * ((float)in / out)), in - 1). */
int dinotrk_mask_upsample(const uint8_t* token_mask, int T, int h, int w, int H, int W, uint8_t* out, void* stream);
/* mask_filter_trajectories (split_trajectories_to_fg_bg.py:55-78) of trajectories traj [N][T][2] (NaN where missing) by
 * masks [Tm][H][W] uint8: a trajectory starts at its first step with both coordinates non-NaN, at (rint(x), rint(y))
 * (torch.round); it is foreground when masks[start][y][x] > 0.  dinotrk_traj_split_count classifies every row, reads the
 * foreground count back to *n_fg (host; synchronises the stream) and returns DINOTRK_EINVAL when a row has no valid step,
 * starts outside the frame or past frame Tm - 1.  dinotrk_traj_split_emit then writes the foreground rows to
 * fg [n_fg][T][2] and the others to bg [N - n_fg][T][2], each in row order. */
size_t dinotrk_traj_split_workspace_bytes(int N);
int dinotrk_traj_split_count(const float* traj, int N, int T, const uint8_t* masks, int Tm, int H, int W, int* n_fg,
                             void* workspace, size_t workspace_bytes, void* stream);
int dinotrk_traj_split_emit(const float* traj, int N, int T, float* fg, float* bg, void* workspace, size_t workspace_bytes,
                            void* stream);

/* ---- best-buddy contrastive losses of the training step (dino_tracker.py:332-344) -------------------------------- */
/* get_bb_pairs_contrastive_loss for all pairs of one loss in one call.  E [N][P][C] is the frame set's token-major
 * embeddings, S / U [B][C] the source / target descriptors of the sampled best buddies; C % 8 == 0.  Group g (host
 * int32 tables) owns rows [grp_row0[g], grp_row0[g] + grp_rows[g]) and the frame slots grp_src[g] / grp_tgt[g]; groups
 * do not overlap, empty groups are skipped, rows of no group are ignored (zero gradient).  cos(a, b) = <a, b> /
 * max(|a| |b|, 1e-8).  Per row r of group g:
 *   out[0][r] = bb = cos(S_r, U_r)
 *   out[1][r] = lse_st = log sum_n exp(cos(S_r, E[t_g][n]) / tau),  out[2][r] = lse_ts (U_r against E[s_g])
 *   out[3][r] = loss_st = lse_st - bb / tau,  out[4][r] = loss_ts = lse_ts - bb / tau
 *   out[5][r] / out[6][r] = the row sums of both cosine rows
 * (out = [7][B] fp32).  The forward keeps the cosines in cos [2B][dinotrk_bb_contrastive_cos_stride(P)] (S rows, then U
 * rows) for the backward.  Cosines run on the split-fp16 wgmma GEMM over copies of E and [S; U] scaled by powers of two
 * (DESIGN.md 3.3): the results do not depend on the inputs' scale.  The backward takes the forward's cos / out and the upstream gradients of loss_st [B], loss_ts [B] and
 * of the per-group means mean_r(bb) and (mean(cos_st) + mean(cos_ts)) / 2 ([n_groups] each); it OVERWRITES dS, dU [B][C]
 * and ADDS the full-frame terms into dE [N][P][C].  Every sum runs in a fixed order: two runs give the same bits.
 * Argument errors (C, frame slots, rows, a short workspace) return DINOTRK_EINVAL before any launch. */
int dinotrk_bb_contrastive_cos_stride(int P);
size_t dinotrk_bb_contrastive_forward_workspace_bytes(int N, int P, int C, int B, int n_groups);
int dinotrk_bb_contrastive_forward(const float* E, int N, int P, int C, const float* S, const float* U, int B,
                                   const int* grp_src, const int* grp_tgt, const int* grp_row0, const int* grp_rows, int n_groups,
                                   float tau, float* cos, float* out, void* workspace, size_t workspace_bytes, void* stream);
/* 0 on invalid arguments */
size_t dinotrk_bb_contrastive_backward_workspace_bytes(int N, int P, int C, int B, const int* grp_src, const int* grp_tgt,
                                                       const int* grp_row0, const int* grp_rows, int n_groups);
int dinotrk_bb_contrastive_backward(const float* E, int N, int P, int C, const float* S, const float* U, int B,
                                    const int* grp_src, const int* grp_tgt, const int* grp_row0, const int* grp_rows,
                                    int n_groups, float tau, const float* cos, const float* out, const float* g_st,
                                    const float* g_ts, const float* g_bbmean, const float* g_cmean, float* dS, float* dU,
                                    float* dE, void* workspace, size_t workspace_bytes, void* stream);

/* ---- training-batch sampler (data/dataset.py:56-258 LongRangeSampler / DinoTrackerSampler) ------------------------ */
/* Trajectories traj [N][T][2] fp32 (NaN where missing).  The sampler stores the valid rows (more than one step with both
 * coordinates non-NaN, dataset.py:100-106) in their order, rows [N'][T][2], and per stored row the bitmask of its valid
 * steps, bits [N'][ceil(T / 32)] uint32 (bit t % 32 of word t / 32).  traj, rows (and gather's rows) may be device or
 * pinned host memory: pinned rows are read and written through the device's mapping, only where needed; pageable host
 * memory is an argument error.  Every element offset is 64-bit; N < 2^31 rows, T <= 65536.  All calls take a workspace
 * of dinotrk_sampler_workspace_bytes(N) bytes; count and select must share it (select reads count's block scan).
 * Argument errors return DINOTRK_EINVAL before any launch.  Profile class "sampler".
 *   prepare_count: *n_valid = N' (host; syncs the stream).  prepare_emit: writes rows [N'] and bits [N'] (no sync).
 *   count: frames [n_frames] int64 are the drawn frame indices (distinct, in [0, T)); a stored row is a candidate when
 *     popcount(bits & frame mask) >= 2 (dataset.py:171).  Writes per-block counts and their scan into the workspace and
 *     reads the total back to *n_cand (host; syncs the stream).
 *   select: for positions perm [m] (< *n_cand, m <= N) among the candidates in row order, row_ids [m] int64 = the stored
 *     row and mat [m][T] fp32 = 1 at the frames that are drawn and valid on that row, else 0 (dataset.py:180-183).  No sync.
 *   gather: t1 / t2 [m][3] = (x, y, t) of rows[row_ids[i]] at steps draws[i][0] / draws[i][1] (draws [m][2] int64, the
 *     multinomial's output; dataset.py:184-188).  No sync. */
size_t dinotrk_sampler_workspace_bytes(int N);
int dinotrk_sampler_prepare_count(const float* traj, int N, int T, int* n_valid, void* workspace, size_t workspace_bytes,
                                  void* stream);
int dinotrk_sampler_prepare_emit(const float* traj, int N, int T, float* rows, uint32_t* bits, void* workspace,
                                 size_t workspace_bytes, void* stream);
int dinotrk_sampler_count(const uint32_t* bits, int N, int T, const int64_t* frames, int n_frames, int* n_cand,
                          void* workspace, size_t workspace_bytes, void* stream);
int dinotrk_sampler_select(const uint32_t* bits, int N, int T, const int64_t* frames, int n_frames, const int64_t* perm,
                           int m, int64_t* row_ids, float* mat, void* workspace, size_t workspace_bytes, void* stream);
int dinotrk_sampler_gather(const float* rows, int T, const int64_t* row_ids, const int64_t* draws, int m, float* t1,
                           float* t2, void* stream);

/* ---- RAFT-large optical flow (torchvision models/optical_flow/raft.py raft_large, eval mode) ---------------------- */
/* Weights: one entry per convolution in torchvision's parameter order.  w_hi / w_lo are the fp16 split
 * (dinotrk_split_fp16) of the K-major matrix [Np][Kp]: row n = output channel, k = (ky * kw + kx) * C_in + ci with the
 * input channels in torchvision's concatenation order, Kp = kh * kw * C_in rounded up to 8, Np = C_out rounded up to
 * 64 (C_out <= 64), 128 (C_out <= 128) or a multiple of 256, padding rows zero; bias [Np] fp32.  Entries 0-15 are the
 * feature encoder (stem, layer1-3 blocks as conv1, conv2 and, for the strided first blocks, the 1 x 1 projection, then
 * the final 1 x 1), 16-31 the context encoder in the same order with its eval-mode BatchNorm folded into weight and
 * bias.  A GRU's convz and convr are ONE entry: the [z; r] matrix with C_out = 256.  scale[i]: a power of two the
 * matrix was divided by before the split (its largest entry in [2^13, 2^14): the fp16 lo halves of small weights would
 * otherwise be subnormal); the GEMM's result is multiplied by it (exact) before the bias is added. */
enum {
  DINOTRK_RAFT_FNET = 0, DINOTRK_RAFT_CNET = 16, DINOTRK_RAFT_CONVCORR1 = 32, DINOTRK_RAFT_CONVCORR2, DINOTRK_RAFT_CONVFLOW1,
  DINOTRK_RAFT_CONVFLOW2, DINOTRK_RAFT_MOTION_CONV, DINOTRK_RAFT_GRU1_ZR, DINOTRK_RAFT_GRU1_Q, DINOTRK_RAFT_GRU2_ZR,
  DINOTRK_RAFT_GRU2_Q, DINOTRK_RAFT_FLOW_HEAD1, DINOTRK_RAFT_FLOW_HEAD2, DINOTRK_RAFT_MASK1, DINOTRK_RAFT_MASK2,
  DINOTRK_RAFT_NCONV
};
typedef struct {
  const void* w_hi[DINOTRK_RAFT_NCONV];
  const void* w_lo[DINOTRK_RAFT_NCONV];
  const float* bias[DINOTRK_RAFT_NCONV];
  float scale[DINOTRK_RAFT_NCONV];
} dinotrk_raft_weights;
/* Frames are [T][3][H][W] fp32 in [0, 1], H, W >= 121 so that the frame replicate-padded to a multiple of 8 (the extra
 * row / column split as torchvision's "sintel" InputPadder) has a 1/8 grid of at least 16 x 16.  Each frame is mapped
 * by 2x - 1 and encoded once: fmap [T][h8 * w8][256] (feature encoder, InstanceNorm statistics in float64 in a fixed
 * order) and, for the first T_ctx frames (the ones flows start from), ctx [T_ctx][h8 * w8][256] = tanh(hidden 128) |
 * relu(context 128) (context encoder; ctx may be NULL when T_ctx = 0).  Workspaces are for one frame size; 0 on invalid
 * arguments. */
size_t dinotrk_raft_encode_workspace_bytes(int H, int W);
int dinotrk_raft_encode(const float* frames, int T, int T_ctx, int H, int W, const dinotrk_raft_weights* w, float* fmap,
                        float* ctx, void* workspace, size_t workspace_bytes, void* stream);
/* Flows [n_pairs][2][H][W] of the pairs (host int32 [n_pairs][2], frames (i, j), the flow i -> j) after
 * num_flow_updates updates: raft_large(frame_i, frame_j, num_flow_updates)[-1], cropped to H x W.  fmap has T frames, ctx
 * the first T_ctx of them (1 <= T_ctx <= T); every j < T and every i < T_ctx, else nothing is launched.  fmap_hi / fmap_lo:
 * the fp16 split of fmap for the correlation volume on the F16X3 GEMM (fp32-faithful inside the split's range, see
 * dinotrk_split_faithful), or both NULL for the exact-fp32 GEMM.  A pair's flow does not depend on the other pairs of
 * the call: the same bits in any batch.  The workspace holds each pair's correlation pyramid (4 * h8 w8 * (h8 w8 + the
 * three pooled levels) bytes) and its update-block activations. */
size_t dinotrk_raft_flow_workspace_bytes(int H, int W, int n_pairs);
int dinotrk_raft_flow(const float* fmap, const void* fmap_hi, const void* fmap_lo, const float* ctx, int T, int T_ctx, int H,
                      int W, const int* pairs, int n_pairs, int num_flow_updates, const dinotrk_raft_weights* w, float* flows,
                      void* workspace, size_t workspace_bytes, void* stream);

/* ---- per-kernel-class device timing (CUDA events on the launching stream; bench.py roofline) ------ */
int dinotrk_profile_classes(void);
const char* dinotrk_profile_class_name(int cls);
void dinotrk_profile_enable(int on);
/* Waits for the recorded events; ms[cls] / launches[cls] accumulate since the previous collect. */
int dinotrk_profile_collect(double* ms, unsigned long long* launches, int n);

/* number of kernel launches issued by this library since load (bench.py's gpu_launches) */
unsigned long long dinotrk_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* DINOTRK_H_ */
