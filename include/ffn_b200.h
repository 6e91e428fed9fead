/*
 * ffn_b200.h — C ABI of libffn_b200.so, the H100-native flood-filling inference engine.
 *
 * This is the boundary a maintainer of google/ffn binds (ctypes stub in INTEGRATION.md) to replace
 * the TensorFlow/JAX executor *and* the numpy flood-fill loop of the inference hot path.  Every
 * entry point names the reference interface it stands in for (paths relative to the reference
 * checkout).  Conventions:
 *
 *   - plain C types only; all coordinates/shapes are (z, y, x), arrays are C-order zyx;
 *   - the caller owns every host buffer, the engine owns every device buffer; handles are opaque;
 *   - every function returns 0 on success, non-zero on failure; ffn_last_error() (thread-local)
 *     describes the failure;
 *   - calls are synchronous; one in-flight call per engine (the Python host serialises);
 *   - there is NO CPU fallback: creation fails if no sm_90 device is usable.
 */
#ifndef FFN_B200_H_
#define FFN_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct FfnEngine FfnEngine;
typedef struct FfnCanvas FfnCanvas;

/* Arithmetic of the 3x3x3 convolutions. */
enum {
  FFN_COMPUTE_FP16_TC = 0, /* fp16 operands, fp32 accumulate on the tensor cores (wgmma); fp32 residual stream */
  FFN_COMPUTE_FP32 = 1,    /* fp32 FMA on CUDA cores ("precise" parity mode) */
  FFN_COMPUTE_FP16X2_TC = 2 /* near-fp32 on the tensor cores: every operand split into fp16 hi + lo parts,
                             * a*w = a_hi*w_hi + a_lo*w_hi + a_hi*w_lo as three wgmma MMAs into the same fp32
                             * accumulator (weights pre-scaled by 2^10 so that w_lo stays normal) */
};

enum { FFN_IMAGE_U8 = 0, FFN_IMAGE_F32 = 1 };

enum { FFN_ARRAY_SEED = 0, FFN_ARRAY_SEGMENTATION = 1, FFN_ARRAY_QPROB = 2, FFN_ARRAY_IMAGE = 3 };

enum { FFN_MASK_MOVEMENT = 0, FFN_MASK_SEED = 1 };

/* Geometry of ConvStack3DFFNModel — ffn/training/models/convstack_3d.py:59-81 (fov_size, deltas,
 * depth, features) with ModelInfo's xyz triples (ffn/training/model.py:25-46) already reversed. */
typedef struct {
  int32_t fov_zyx[3];
  int32_t deltas_zyx[3];
  int32_t depth;    /* residual modules; 2*depth 3x3x3 convolutions + conv_lom */
  int32_t features; /* must be 32 */
} FfnModelDesc;

/* InferenceOptions (ffn/inference/inference.proto:131-168) after Canvas.__init__ converted the
 * probabilities to logits and stored them back as float32 (ffn/inference/inference.py:186-195),
 * plus the float64 movement-policy threshold of movement.get_policy_fn (movement.py:241-242). */
typedef struct {
  float init_activation;        /* logit */
  float pad_value;              /* logit */
  float move_threshold;         /* logit, float32 — Canvas.is_valid_pos / disco test */
  float segment_threshold;      /* logit */
  float disco_seed_threshold;   /* probability-space fraction; < 0 disables (inference.py:416) */
  double policy_score_threshold;/* FaceMaxMovementPolicy.score_threshold (float64 logit) */
  int32_t min_boundary_dist_zyx[3];
  int32_t min_segment_size;
} FfnOptions;

/* Result of one Canvas.segment_at (ffn/inference/inference.py:460-533). */
typedef struct {
  int64_t iters;            /* return value of segment_at */
  int32_t min_pos[3];       /* Canvas._min_pos */
  int32_t max_pos[3];       /* Canvas._max_pos */
  int32_t seed_got_too_weak;
  int32_t queue_len;        /* entries left in the movement-policy deque */
  int32_t finished;         /* 0 if max_steps was hit before the queue drained (call again to resume) */
  int32_t reserved;
} FfnSegStats;

/* storage.OriginInfo (ffn/inference/storage.py:35) per accepted segment. */
typedef struct {
  int32_t id;
  int32_t start_zyx[3];
  int64_t iters;
  double walltime_sec;
} FfnOrigin;

/* One (segment, overlapped id, voxel count) triple of Canvas.overlaps (inference.py:624-632,668). */
typedef struct {
  int32_t id;
  int32_t other_id;
  int64_t count;
} FfnOverlap;

/* Counters named as in ffn/inference/inference.py (counters['...']). */
typedef struct {
  int64_t inference_calls;      /* 'inference-calls' == FoV steps */
  int64_t segment_at_calls;     /* 'segment_at-loop-calls' */
  int64_t seeds_examined;       /* seeds that reached Canvas (after the border filter of seed.py:81-88) */
  int64_t skip_threshold;
  int64_t skip_invalid_pos;
  int64_t skip_restricted_pos;  /* 'skip_restriced_pos' (sic) */
  int64_t seed_got_too_weak;
  int64_t voxels_segmented;
  int64_t voxels_overlapping;
  int64_t invalid_weak;         /* segments rejected: weak seed */
  int64_t invalid_small;        /* segments rejected: too small */
  int64_t invalid_other;        /* segments rejected: num_iters <= 0 */
  int64_t segments;             /* accepted */
  int64_t max_id;               /* Canvas._max_id */
  double device_seconds;        /* sum of kernel time (CUDA events) of this call */
  int64_t kernel_launches;
} FfnCounters;

const char* ffn_last_error(void);

/* ---- engine: owns device context, packed weights, workspace ------------------------------
 * Replaces Runner._init_tf_model + Saver.restore (ffn/inference/runner.py:98-163).
 * weights_dhwio[i]: float32 [3,3,3,Cin,32] in TF DHWIO order for i < 2*depth (Cin = 2 for i == 0),
 * weights_dhwio[2*depth]: conv_lom [1,1,1,32,1]; biases[i]: [32] (conv_lom: [1]). */
int ffn_engine_create(int device, const FfnModelDesc* model, const float* const* weights_dhwio,
                      const float* const* biases, int compute_mode, FfnEngine** out);
/* Canvases created from the engine may outlive this call: the engine is then released by the last
 * ffn_canvas_destroy (until then those canvases stay fully usable). */
void ffn_engine_destroy(FfnEngine* engine);
int ffn_engine_set_compute_mode(FfnEngine* engine, int compute_mode);
/* Flood-fill chains time-multiplexed over the SMs by ONE persistent kernel (1..4; 0 = default 4): objects of a
 * canvas in flight at once in ffn_canvas_segment_all (committed in seed order — the results are those of the
 * sequential reference loop, inference.py:538-683, for any value), and patches of a batch sharing a round in
 * ffn_predict (the reference batches FoVs into one session.run, executor.py:266-340).  1 = strictly one
 * object / patch at a time. */
int ffn_engine_set_chains(FfnEngine* engine, int max_chains);
/* FoV steps one launch of the persistent kernel may run in ffn_canvas_segment_at / ffn_canvas_segment_all before it
 * pauses at a round boundary and the host launches it again (0 = the default, 2^15).  A small chunk makes every
 * object cross launch boundaries: the results do not depend on it. */
int ffn_engine_set_step_chunk(FfnEngine* engine, int64_t steps);
/* Number of SMs (CTAs of the cooperative grid) this engine's kernel occupies; 0 = all.  Several engines
 * with disjoint SM budgets (e.g. 3 x 44) driven from different host threads run their persistent kernels
 * CONCURRENTLY on one GPU: the H100 form of the reference's batching across canvases
 * (InferenceRequest.batch_size / concurrent_requests, doc/manual.md:89-97). */
int ffn_engine_set_grid(FfnEngine* engine, int num_ctas);
/* sm count, cooperative grid size, shared memory per CTA, tiles per FoV: info[0..3]. */
int ffn_engine_info(FfnEngine* engine, int64_t info[8]);

/* Device-side cycle counters of CTA 0 (out[0..31]) and the last CTA (out[32..63]): slot 0 grid-barrier
 * wait, 1 activation TMA wait, 2 weight wait, 3 MMAs (issue to completion), 4 unused, 5 epilogue body,
 * 6 stage, 7 paste, 8 leader, 9 steps, 10 kernel, 11 conv layers, 12 leader policy (queue pushes + pops), 13 pops,
 * 14 chain-barrier wait, 15 unused; the leader by phase: 16 state copy-in + the face maxima, (12: policy
 * updates + pops), 17 scheduler (chain_advance), 18 state copy-out + release; 19 wait for the leader's round flag,
 * 20 face reduce; 21-31 unused.
 * Off by default (reading the clock perturbs the critical CTA): ffn_engine_profile(e, NULL, 1) switches
 * the counters on, (e, NULL, 0) off; with out != NULL the counters are returned (and reset if reset). */
int ffn_engine_profile(FfnEngine* engine, int64_t out[64], int reset);
/* The table the flood kernel reduces the movement policy's six faces from (host only, no device needed): the face
 * voxels of `model`'s field of view ordered by the kernel's row index, entries[3 i ..] = (row, face = 2 * axis +
 * (positive side), C-order index inside the face); at most `cap` entries are written (entries may be NULL), their
 * number goes to *n_entries.  tile_first (NULL or [*n_tiles + 1], call once to learn *n_tiles): first entry of every
 * 126-row tile.  Debug / tests. */
int ffn_face_table(const FfnModelDesc* model, int64_t cap, int32_t* entries, int64_t* n_entries, int32_t* tile_first,
                   int64_t* n_tiles);
/* Tile timeline of one CTA (CTA 1) recorded while the counters are on: out[e * 2048 + i] = SM clock when event e
 * happened to that role's i-th tile since kernel start (0 producer saw the chain barrier, 1 copies issued,
 * 2 consumers saw the operands, 4 MMAs complete, 6 epilogue done, 7 i-th barrier release by the signal warp; 3 and
 * 5 are not recorded); 0 = not recorded.  n <= 8 * 2048.  Debug only. */
int ffn_engine_trace(FfnEngine* engine, int64_t* out, int64_t n, int reset);

/* ---- L0 drop-in: ExecutorClient.predict (ffn/inference/executor.py:134-139, 266-340) -------
 * seed, image: host float32 [batch, Z, Y, X]; logits_out: host float32 [batch, Z, Y, X]
 * (the 'logits' fetch without the trailing channel axis).  Copies in, runs, copies out. */
int ffn_predict(FfnEngine* engine, const float* seed, const float* image, int batch,
                float* logits_out);

/* ---- canvas: HBM-resident state of ffn.inference.inference.Canvas (inference.py:129-310) ---
 * image: host [Z,Y,X] uint8 (normalised on the fly as (x - mean) / stddev in float32, exactly
 * runner.py:383-385) or float32 (already normalised; mean/stddev ignored). */
int ffn_canvas_create(FfnEngine* engine, const void* image, int image_dtype,
                      const int32_t shape_zyx[3], float image_mean, float image_stddev,
                      const FfnOptions* options, int keep_probability_maps, FfnCanvas** out);
void ffn_canvas_destroy(FfnCanvas* canvas);
/* MovementRestrictor.mask / .seed_mask (movement.py:290-314); mask: host uint8 [Z,Y,X] or NULL. */
int ffn_canvas_set_mask(FfnCanvas* canvas, int which, const uint8_t* mask);

/* Canvas.segment_at (inference.py:460-533).  reset == 1: init_seed + reset_state first
 * (partial_segment_iters == 0 path); reset == 2: reset_state only — the seed and the extents are kept
 * (Canvas.reset_seed_per_segment == False, inference.py:486-490); reset == 0 resumes the current object.  Runs at most
 * max_steps FoV steps (<= 0: unlimited) inside ONE persistent kernel launch per ~budget. */
int ffn_canvas_segment_at(FfnCanvas* canvas, const int32_t start_zyx[3], int reset,
                          int64_t max_steps, FfnSegStats* out);

/* Canvas.segment_all (inference.py:538-683) over an explicit seed list (the coords a seed policy
 * produced, seed.py:63-95).  origins_out / overlaps_out: caller arrays with the given capacities;
 * n_origins / n_overlaps receive the counts (ids are assigned as ++max_id in seed order). */
int ffn_canvas_segment_all(FfnCanvas* canvas, const int32_t* seeds_zyx, int64_t n_seeds,
                           FfnOrigin* origins_out, int64_t origins_cap, int64_t* n_origins,
                           FfnOverlap* overlaps_out, int64_t overlaps_cap, int64_t* n_overlaps,
                           FfnCounters* counters_out);

/* Canvas.update_at (inference.py:386-441): one FoV step at pos, no movement policy.
 * pred_out: host float32 [Z,Y,X] of the FoV (the merged logits pasted into the seed). */
int ffn_canvas_update_at(FfnCanvas* canvas, const int32_t pos_zyx[3], float* pred_out);

/* Canvas.init_seed (inference.py:443-450). */
int ffn_canvas_init_seed(FfnCanvas* canvas, const int32_t pos_zyx[3]);

/* Lazy views of Canvas.seed / .segmentation / .seg_prob (and the image as float32): copy a box. */
int ffn_canvas_read(FfnCanvas* canvas, int which, const int32_t lo_zyx[3],
                    const int32_t size_zyx[3], void* dst);
int ffn_canvas_write(FfnCanvas* canvas, int which, const int32_t lo_zyx[3],
                     const int32_t size_zyx[3], const void* src);

/* Movement-policy state for .cpoint compatibility (movement.py:180-184): deque entries as
 * (score, z, y, x) float64 quadruples, done-set as int32 lattice triples, start position. */
int ffn_canvas_policy_state_size(FfnCanvas* canvas, int64_t* queue_len, int64_t* done_len);
int ffn_canvas_policy_state_get(FfnCanvas* canvas, double* queue_szyx, int32_t* done_zyx,
                                int32_t start_zyx[3]);
int ffn_canvas_policy_state_set(FfnCanvas* canvas, const double* queue_szyx, int64_t queue_len,
                                const int32_t* done_zyx, int64_t done_len,
                                const int32_t start_zyx[3]);
/* Resume of an in-flight object restored from a .cpoint (Canvas.restore_checkpoint returning
 * partial_segment_iters > 0, inference.py:728-778): after ffn_canvas_policy_state_set and the
 * seed/segmentation writes, the next ffn_canvas_segment_all first finishes this object (with
 * the given iteration count and extents) and commits it, then continues with its seed list. */
int ffn_canvas_set_resume(FfnCanvas* canvas, int64_t iters, const int32_t min_pos[3],
                          const int32_t max_pos[3]);
/* Event log of the device loop (debugging, Canvas.history export).  Call with capacity > 0 and
 * events_out == NULL to (re)start logging, capacity == 0 to stop; call with events_out != NULL to
 * fetch: rows of (type, z, y, x), type 1 push, 2 pop valid, 3 pop invalid, 4 pop below threshold,
 * 5 pop already done, 6 FoV step, 7 seed invalid, 8 object start, 9 (count, 0, 0) = Canvas.history_deleted of the step just
 * executed (inference.py:420-422).  *n_events = events produced (may exceed capacity). */
int ffn_canvas_trace(FfnCanvas* canvas, int64_t capacity, int32_t* events_out, int64_t* n_events);
/* PolicyPeaks on the device (ffn/inference/seed.py:142-199): Sobel magnitude -> gaussian(sigma 49/6)
 * adaptive threshold -> exact Euclidean distance transform (anisotropy = voxel size) -> local maxima
 * (min_distance 3) with the tie-break noise `noise` (host float64 [Z,Y,X] = RandomState(42).rand, or
 * NULL).  Uses the canvas' resident image, segmentation and masks.  coords_out receives up to `cap`
 * (z, y, x) triples in arbitrary order (sort them for the policy); *n_out = number of peaks found. */
int ffn_canvas_seed_peaks(FfnCanvas* canvas, const float voxel_size_zyx[3], const double* noise,
                          int32_t* coords_out, int64_t cap, int64_t* n_out);

/* Seed policies built on peak_local_max (ffn/inference/seed.py:133-139, 202-352). */
enum {
  FFN_SEED_PEAKS_2D = 0,   /* PolicyPeaks2d: per z-slice 2-D Sobel -> gaussian(sigma 49/6) threshold, movement mask as
                            * edges -> unit-spacing 2-D EDT; peaks within each slice; noise [Y,X] */
  FFN_SEED_FILL_EMPTY = 1, /* PolicyFillEmptySpace: 3-D EDT of segmentation == 0; noise [Z,Y,X] */
  FFN_SEED_MAX_PEAKS = 2   /* PolicyMaxPeaks: image with labels > 0 | movement mask | seed mask set to 0; noise [Z,Y,X] */
};
typedef struct {
  int32_t kind;                 /* FFN_SEED_* */
  int32_t min_distance;         /* neighbourhood radius and border exclusion (y, x; and z unless PEAKS_2D) */
  double threshold_abs;
  int32_t threshold_abs_is_min; /* threshold_abs=None: the minimum key */
  int32_t use_threshold_rel;    /* 0: threshold_rel=None */
  double threshold_rel;         /* threshold = max(threshold_abs, threshold_rel * maximum key) */
} FfnSeedPolicyDesc;
/* The peaks of one of the policies above on the canvas' resident image, segmentation and masks: voxels whose
 * key (double)value + noise * 1e-4 (noise: host float64 = RandomState(42).rand, or NULL) equals the maximum of
 * its (2 min_distance + 1)-box (edges clamped), exceeds the threshold and lies min_distance or more from the
 * border.  A slice (PEAKS_2D) or canvas (FILL_EMPTY) without any background voxel for the distance transform
 * has no finite distance and yields no peaks.  coords_out / cap / *n_out as for ffn_canvas_seed_peaks. */
int ffn_canvas_seed_policy(FfnCanvas* canvas, const FfnSeedPolicyDesc* desc, const double* noise,
                           int32_t* coords_out, int64_t cap, int64_t* n_out);
/* Canvas._max_id / counters carried across calls (checkpoint restore, init segmentation). */
int ffn_canvas_set_max_id(FfnCanvas* canvas, int64_t max_id);
int ffn_canvas_get_counters(FfnCanvas* canvas, FfnCounters* out);
/* Bookkeeping of the last ffn_canvas_segment_all: out[0] objects started ahead of their turn, out[1] of
 * those discarded (re-run in turn or rejected by the in-order gating), out[2] FoV steps of the discarded runs,
 * out[3] FoV steps executed in total (FfnCounters.inference_calls counts only what the reference counts),
 * out[4] rounds of the persistent kernel, out[5] / out[6] chain-rounds spent without an object / waiting for the
 * turn to commit, out[7] chains used. */
int ffn_canvas_spec_stats(FfnCanvas* canvas, int64_t out[8]);
/* Scheduler transitions of the last ffn_canvas_segment_all, out[0 .. n) (17 values; unused slots are set to 0):
 * [0] finished objects parked to wait for their turn, [1] runs suspended so that a parked object could commit,
 * [2] suspended runs resumed, [3] chain-rounds a run suspended in that same round had to wait before it could go on
 * (its last paste was still landing), [4] parked objects taken up at their turn, [5] early runs validated, [6] / [7]
 * early runs discarded and their seed rejected / redone in turn ([6] + [7] == spec_stats out[1]), [8] conflicts found
 * only among the popped-but-not-stepped trajectory entries, [9] / [10] early runs validated / discarded with such
 * entries, [11] chain-rounds idle because every buffer of the chain was in use, [12] moves of Canvas.seed's last
 * in-turn object to the snapshot array, [13] seeds skipped at the head of the line because no buffer held them (never
 * expected), [14] kernel launches, [15] / [16] launches that paused with a parked or suspended object / with a commit
 * under way. */
int ffn_canvas_sched_stats(FfnCanvas* canvas, int64_t* out, int n);

/* Multi-GPU merge helpers (SURVEY.md 8e): raw device pointers for NCCL, and the HBM-bound
 * relabel kernel that adds a rank's ID offset to every label > 0. */
int ffn_canvas_device_ptr(FfnCanvas* canvas, int which, void** ptr, int64_t* bytes);
int ffn_canvas_add_id_offset(FfnCanvas* canvas, int32_t offset);

/* ---- decision points: find_decision_points (ffn/utils/decision_point.py:27-145) ---------------------------------
 * Every empty voxel takes the id of the nearest labelled voxel (exact squared physical distance; the smallest id
 * on ties), unless that distance exceeds max_distance.  Within the box, every pair of different ids (a < b) that
 * then touch under one of the 7 offsets of itertools.product((0,-1),(0,-1),(0,-1)) gets the minimal
 * dist = (edt_a + edt_b) / 2 and, among the rows at that minimum, the one closest to their centroid (first in
 * (offset, raster) order on ties). */
typedef struct {
  int32_t shape_zyx[3];
  int32_t voxel_size_xyz[3];  /* positive integers */
  int32_t use_max_distance;   /* 0: max_distance=None */
  int32_t reserved;
  double max_distance;
  int32_t box_start_zyx[3];   /* subvol_box; the whole volume when it is not given */
  int32_t box_size_zyx[3];
  int64_t dust_threshold;     /* > 0: clear_dust first, ids with fewer voxels become 0 (optimize_sparse) */
} FfnDecisionPointDesc;
typedef struct {
  uint64_t id_a, id_b;        /* id_a < id_b */
  double dist;
  int64_t point_xyz[3];       /* relative to the box */
} FfnDecisionPoint;
/* labels: host uint64 [Z,Y,X]; written back (dust cleared) only when dust_threshold removed an id.  out receives the
 * first min(count, cap) decision points in (id_a, id_b) order; *n_out = count.  Fails, with no approximate answer,
 * when (D_max + 1) * M does not fit in 64 bits (D_max: the largest squared physical distance in the volume, M: the
 * power of two above the number of ids). */
int ffn_decision_points(int device, const FfnDecisionPointDesc* desc, uint64_t* labels, FfnDecisionPoint* out,
                        int64_t cap, int64_t* n_out);

/* ---- resegmentation analysis: evaluate_{pair,endpoint}_resegmentation (ffn/inference/resegmentation_analysis.py:97-260)
 * A batch of items of one kind whose boxes all have the extent box_zyx, laid out back to back (item-major, C-order
 * zyx): labels [n][box] uint64 original ids, probs [n][2][box] (pair: the analysis box of both objects) or [n][1][box]
 * (endpoint: the whole segmentation box) uint8 quantised probabilities, ids [n][2] (id_a, id_b; id_b unused for an
 * endpoint).  A voxel belongs to a resegmented object where mask_table[q] != 0; the caller builds the table from its
 * own dequantisation and threshold comparison. */
typedef struct {
  int32_t box_zyx[3];
  int32_t voxel_size_zyx[3];  /* positive integers; pairs only */
  int32_t pair;               /* 1: pair items, 0: endpoint items */
  int32_t reserved;
  int64_t num_items;
} FfnResegEvalDesc;
/* Per item.  seg_k = (label == id of object k), reseg_k = mask of probability box k.  max_edt2: the largest exact
 * squared physical distance to the nearest voxel outside the mask (scipy's distance_transform_edt squared) of seg_0,
 * seg_1, reseg_0, reseg_1; 0 for an empty mask.  A mask without any voxel outside it in the box gets what scipy
 * returns there, (Z wz)^2 + ((Y-1) wy)^2 + ((X-1) wx)^2.  Endpoint items fill n_seg[0] and n_reseg[0] only. */
typedef struct {
  int64_t n_seg[2];
  int64_t n_reseg[2];
  int64_t n_reseg_seg[2][2];  /* [k][j] = |reseg_k & seg_j| */
  int64_t n_inter, n_union;   /* |reseg_0 & reseg_1|, |reseg_0 | reseg_1| */
  uint64_t max_edt2[4];
} FfnResegStats;
/* Endpoint items: one row per (item, original id) with num_overlapping > 0, in (item, id) order; id 0 included. */
typedef struct {
  int64_t item;
  uint64_t id;
  int64_t num_overlapping;    /* voxels of the id inside the mask */
  int64_t num_original;       /* voxels of the id in the box */
} FfnResegOverlap;
/* stats_out: [n].  overlaps_out receives the first min(count, cap) rows; *n_overlaps = count (0 for pairs).  Fails
 * when a squared distance could reach 2^63, or when the batch holds 2^31 or more mask voxels (four masks per pair item). */
int ffn_reseg_eval(int device, const FfnResegEvalDesc* desc, const uint64_t* labels, const uint8_t* probs,
                   const uint64_t* ids, const uint8_t mask_table[256], FfnResegStats* stats_out,
                   FfnResegOverlap* overlaps_out, int64_t cap, int64_t* n_overlaps);

/* ---- split consensus: split_segmentation_by_intersection (ffn/inference/segmentation.py:181-290) ----------------
 * a, b: host uint64 [n] label arrays of the same shape.  Every overlapping pair (id_a, id_b), in (id_b, id_a) order,
 * maps to 0 when it has fewer than min_size voxels or id_a == 0; to id_a when id_b is id_a's largest overlap (the
 * smallest id_b on equal counts); otherwise to the next new id max(a) + 1, max(a) + 2, ...  a is rewritten in place
 * with the pair ids; b is only read.  Fails, with no approximate answer, when n >= 2^31 or when max(a) plus the number
 * of new ids does not fit in 64 bits. */
int ffn_split_intersection(int device, int64_t n, uint64_t* a, const uint64_t* b, int64_t min_size);

/* ---- partition map: compute_partitions (compute_partitions.py:115-204) -------------------------------------------
 * Exclusion sphere, with the values as given: voxel (x, y, z) of the volume is inside when
 * (x - cx)^2 + (y - cy)^2 + (z - cz)^2 <= r2, in wrapping int64 (c_xyz, r2) when `integer`, else in float64 (f_xyz,
 * f_r2) summed left to right. */
typedef struct {
  int64_t c_xyz[3];
  int64_t r2;
  double f_xyz[3];
  double f_r2;
  int32_t integer;
  int32_t reserved;
} FfnExclusionSphere;
typedef struct {
  int32_t shape_zyx[3];
  int32_t lom_radius_zyx[3];
  int64_t min_size;              /* non-zero ids with fewer voxels are cleared first (written back); <= 0: none */
  const double* thresholds;      /* [n_thresholds], in list order */
  int32_t n_thresholds;
  int32_t use_whitelist;         /* 1: only ids in whitelist[] are partitioned */
  const uint64_t* whitelist;     /* [n_whitelist] ids, signed ids by their two's-complement bits */
  int64_t n_whitelist;
  const FfnExclusionSphere* spheres;
  int32_t n_spheres;
  int32_t reserved;
  int64_t scratch_bytes;         /* count scratch per group of labels (8 B per grown-box voxel); <= 0: a quarter of
                                  * the free device memory.  A label larger than the budget gets a group of its own. */
  int64_t* n_labels_out;         /* optional: the number of labels partitioned (kept after dust and whitelist) */
} FfnPartitionDesc;
/* labels: host uint64 [z][y][x], rewritten in place when dust is cleared.  mask: host uint8 [z][y][x] (non-zero =
 * masked) or NULL.  out: host uint8 [(z - 2 rz)][(y - 2 ry)][(x - 2 rx)] (the VALID region; nothing when an extent is
 * not positive): 255 where the LOM box holds a masked voxel or the voxel lies in an exclusion sphere; else, at a voxel
 * of a partitioned label, i + 1 for the first i with count / prod(2r + 1) < thresholds[i] (float64), or
 * n_thresholds + 1; else 0.  counts: the 256-bin histogram of out.  Fails, with no approximate answer, for 2^31 or
 * more voxels or a negative radius. */
int ffn_compute_partitions(int device, const FfnPartitionDesc* desc, uint64_t* labels, const uint8_t* mask,
                           uint8_t* out, int64_t counts[256]);

/* ---- training coordinates: build_coordinates (build_coordinates.py:61-112) -----------------------------------------
 * One crop of a partition volume: volume[start + (0 .. crop_shape)] on every axis (z, y, x). */
typedef struct {
  int32_t shape_zyx[3];          /* the uint8 volume, C order */
  int32_t crop_start_zyx[3];
  int32_t crop_shape_zyx[3];     /* fewer than 2^31 voxels in all; an empty crop writes nothing */
  int32_t reserved;
  int64_t volume_index;          /* written as the first element of every row */
} FfnPartitionRowsDesc;
/* volume: host uint8 [z][y][x].  rows: host int64 [crop voxels][2], of which the first (crop voxels - counts[255])
 * are written: (volume_index, flat crop index) for every voxel whose value is not 255, grouped by value in ascending
 * order and in ascending flat order within a value.  counts: the 256-bin histogram of the crop. */
int ffn_partition_rows(int device, const FfnPartitionRowsDesc* desc, const uint8_t* volume, int64_t* rows,
                       int64_t counts[256]);

/* One volume of the coordinate records: center = margin + unravel(flat, crop_shape), reversed to (x, y, z). */
typedef struct {
  int32_t crop_shape_zyx[3];
  int32_t margin_zyx[3];         /* not negative */
  int64_t name_offset;           /* label_volume_name: names[name_offset .. + name_length] */
  int64_t name_length;
} FfnCoordinateVolume;
typedef struct {
  const FfnCoordinateVolume* volumes;
  int32_t n_volumes;
  int32_t reserved;
  const uint8_t* names;
  int64_t names_bytes;
} FfnCoordinateDesc;
/* rows: host int64 [n_rows][2] of (volume, flat crop index).  out: host bytes [out_capacity]; receives, per row in
 * order, the TFRecord frame (u64 length | u32 masked CRC-32C | payload | u32 masked CRC-32C, as TFRecordWriter writes
 * it before compression) of tf.train.Example {center: Int64List [x, y, z], label_volume_name: BytesList [name]} in
 * protobuf's deterministic encoding.  *out_bytes: the bytes written.  Fails for a row outside the volume table or an
 * out_capacity below the frames' size (*out_bytes then holds the size needed). */
int ffn_coordinate_records(int device, const FfnCoordinateDesc* desc, const int64_t* rows, int64_t n_rows,
                           uint8_t* out, int64_t out_capacity, int64_t* out_bytes);

/* ---- connected components: clean_up / clean_up_and_count (ffn/inference/segmentation.py:89-178) ------------------
 * A component is a maximal set of voxels of one non-zero id connected under 6- (1), 18- (2) or 26-connectivity (3).
 * Components are numbered 1, 2, ... in C order of their first voxel; 0 stays 0.  Then every component with fewer than
 * min_size voxels becomes 0 (its number stays unused). */
typedef struct {
  int32_t shape_zyx[3];
  int32_t connectivity;   /* 1, 2 or 3 */
  int64_t min_size;       /* <= 0: no size filter */
} FfnCleanUpDesc;
/* labels: host uint64 [z][y][x], rewritten in place with the component numbers.  Table (ids, orig_ids, counts, each
 * optional; all NULL with cap = 0 when no table is wanted): one row per output id in ascending order, 0 first when the
 * output has a 0: the id, the input id at the id's first voxel in the output, and its voxel count.  *n_ids: the rows.
 * When a table is wanted and *n_ids > cap, nothing is written, labels included: call again with cap = *n_ids.  Fails
 * for 2^31 or more voxels, a negative extent or a connectivity other than 1, 2, 3. */
int ffn_clean_up(int device, const FfnCleanUpDesc* desc, uint64_t* labels, uint64_t* ids, uint64_t* orig_ids,
                 int64_t* counts, int64_t cap, int64_t* n_ids);

/* ---- training step: train.py:135-152 with model.py:115-157 and optimizer.py:73-112 ---------------------------------
 * One sess.run([train_op, global_step, logits]) of the reference's train.py on a batch of field-of-view patches:
 * forward pass, mean(sigmoid_cross_entropy_with_logits(logits, labels) * loss_weights) over all batch * Z * Y * X
 * elements, backward pass, every gradient entry clipped to +-max_gradient_entry_mag, one optimizer step.  The 3x3x3
 * convolutions run on the tensor cores with bf16 operands and fp32 accumulation; the residual stream, conv_lom, the
 * weights, biases and optimizer slots are fp32.  Every reduction runs in a fixed order: two identical steps give
 * bit-identical weights. */
typedef struct FfnTrainer FfnTrainer;
enum { FFN_OPT_SGD = 0, FFN_OPT_MOMENTUM = 1, FFN_OPT_ADAM = 2 };
typedef struct {
  int32_t optimizer;              /* FFN_OPT_* */
  float momentum;                 /* momentum: MomentumOptimizer's momentum (not Nesterov) */
  float beta1, beta2, epsilon;    /* adam: AdamOptimizer's beta1, beta2, epsilon */
  float max_gradient_entry_mag;   /* <= 0: no clipping */
  int32_t max_batch;              /* patches per call the trainer allocates for */
} FfnTrainDesc;
/* weights_dhwio / biases as for ffn_engine_create; the model checks are those of ffn_engine_create.  The trainer keeps
 * its own fp32 copy of the weights and the optimizer slots (zero), and owns all its device memory. */
int ffn_trainer_create(int device, const FfnModelDesc* model, const float* const* weights_dhwio,
                       const float* const* biases, const FfnTrainDesc* desc, FfnTrainer** out);
void ffn_trainer_destroy(FfnTrainer* trainer);
/* seed, image, labels, loss_weights (NULL: all 1): host float32 [batch, Z, Y, X], 1 <= batch <= max_batch.  Runs the
 * step at learning_rate (the host applies any decay) and advances the global step.  logits_out (NULL: not returned):
 * the logits of the weights before the update.  *loss_out: the loss, summed in float64. */
int ffn_trainer_step(FfnTrainer* trainer, const float* seed, const float* image, const float* labels,
                     const float* loss_weights, int batch, float learning_rate, float* logits_out, double* loss_out);
/* The same forward and backward pass without the update: d loss / d logits [batch, Z, Y, X] and the raw (unclipped)
 * gradients in the layout of weights_dhwio / biases (any pointer may be NULL).  Changes nothing. */
int ffn_trainer_gradients(FfnTrainer* trainer, const float* seed, const float* image, const float* labels,
                          const float* loss_weights, int batch, float* dlogits_out, float* const* weight_grads,
                          float* const* bias_grads, double* loss_out);
/* The current weights in the layout ffn_engine_create takes, and the number of steps run. */
int ffn_trainer_get_weights(FfnTrainer* trainer, float* const* weights_dhwio, float* const* biases,
                            int64_t* global_step);

/* ---- training examples: train.py:202-286, 353-412 and ffn/training/examples.py ------------------------------------
 * The example loop of the reference's train.py, resident on the device: per batch element a training patch (image,
 * softened labels and the seed canvas, each fov + 2 * deltas * moves voxels per axis, with moves = fov_moves for the
 * fixed policy and fov_moves + 1 for max_pred_moves), the offset of its field of view and the state of its move policy.
 * One step pastes the previous step's logits into the seed, resumes the policy on the updated seed and, when it is
 * exhausted, loads the next example of the coordinate stream (crop, object mask of the centre label, 0.95 / 0.05
 * labels, the example's axis permutation and reflections, (image - offset) / scale in float32).  New examples go to
 * the elements in element order 0 .. batch-1 within a step.  A fresh example always yields its centre, so an element
 * takes at most one new example per step. */
typedef struct FfnExamples FfnExamples;
enum { FFN_FOV_FIXED = 0, FFN_FOV_MAX_PRED_MOVES = 1 };
typedef struct {
  int32_t volume;                 /* index into the volumes given to ffn_examples_create */
  int32_t center_xyz[3];          /* the crop is centre - (size - 1) // 2 .. + size */
  int32_t permutation_zyx[3];     /* axis i of the example is axis permutation_zyx[i] of the crop (np.transpose) */
  int32_t reflect_zyx[3];         /* nonzero: that axis is reversed after the permutation */
} FfnExampleCoord;
typedef struct {
  const uint8_t* image;           /* host [z][y][x] */
  const int64_t* labels;          /* host [z][y][x]; ids <= 0 are background */
  int32_t image_shape_zyx[3];
  int32_t label_shape_zyx[3];
  float offset, scale;            /* image normalisation of this volume */
} FfnExampleVolume;
typedef struct {
  int32_t policy;                 /* FFN_FOV_* */
  int32_t fov_moves;              /* >= 1 */
  float seed_pad;                 /* in (0, 1) */
  float seed_logit_pad;           /* float32 logit(seed_pad) and logit(0.95) of the fresh seed, as the host computes */
  float seed_logit_centre;        /*   them (scipy.special.logit on float32) */
  int32_t batch;
  double seed_threshold;          /* logit(threshold): a move's target is valid when seed >= it, compared in float64 */
  double label_threshold;         /* expit(logit(threshold)): wanted when label >= it (max_pred_moves), in float64 */
  const int32_t* shifts_zyx;      /* fixed: [n_shifts][3], the visiting order after the centre */
  int32_t n_shifts;
  int32_t permutable_zyx[3];      /* nonzero: the axis may be permuted (all such axes need equal patch extents) */
  int32_t reflectable_zyx[3];     /* nonzero: the axis may be reflected */
  double eval_threshold;          /* the tracker's logit(0.9) (scipy's value): a voxel is predicted when seed >= it */
} FfnExampleDesc;
/* model: the fov and deltas of the network trained (the trainer's).  The volumes are copied to the device.  Fails
 * for seed_pad outside (0, 1), a fresh seed whose centre fails seed_threshold, permutable axes of unequal patch extent,
 * a batch outside [1, 32], fov_moves < 1 or patches of 2^31 or more voxels.  The object owns all its device memory. */
int ffn_examples_create(int device, const FfnModelDesc* model, const FfnExampleDesc* desc,
                        const FfnExampleVolume* volumes, int n_volumes, FfnExamples** out);
void ffn_examples_destroy(FfnExamples* examples);
/* One step of the loop without training: coords are the next n_coords entries of the example stream (at least
 * batch).  Writes the batch (seed, image, labels: host float32 [batch, Z, Y, X]; any may be NULL), each element's
 * offset (z, y, x) from its patch centre and index of its example in the stream since creation, and the entries
 * taken.  Fails, changing nothing, for a coordinate whose crop leaves its volume, an unknown volume or a permutation or
 * reflection of an axis the description does not allow. */
int ffn_examples_next(FfnExamples* examples, const FfnExampleCoord* coords, int64_t n_coords, float* seed_out,
                      float* image_out, float* labels_out, int32_t* offsets_zyx_out, int64_t* example_out,
                      int64_t* n_consumed);
/* Pastes logits (host float32 [batch, Z, Y, X]) into each element's seed at its current offset. */
int ffn_examples_update(FfnExamples* examples, const float* logits);
/* The seed canvases, host float32 [batch, patch z, y, x]. */
int ffn_examples_read_seeds(FfnExamples* examples, float* out);
/* The tracker of the loop (ffn/training/tracker.py's EvalTracker, as examples.py feeds it), kept on the device by
 * every step of ffn_examples_next and ffn_trainer_train.  Moves: every move the policy evaluates, as record_move
 * counts them, at radius int(|shift|) for fixed and 0 for max_pred_moves; the centre move of each new example counts.
 * Finished examples (add_patch): on the crop of fov + 2 * deltas * fov_moves voxels at the patch centre, TP / TN /
 * FP / FN of (seed >= eval_threshold, label > 0.5) and the mean sigmoid cross-entropy
 * max(x, 0) - x z + log1p(exp(-|x|)) in float64, and the centre planes of the last 16 of them. */
typedef struct {
  int64_t steps;                  /* loop steps */
  int64_t patches;                /* finished examples */
  int64_t eval_voxels;            /* voxels of their eval crops */
  int64_t prediction_counts[4];   /* TP, TN, FP, FN */
  double patch_loss;              /* sum of the finished examples' mean losses, in finishing order */
} FfnTrackerCounts;
/* Reads the counts since the last reset.  moves_by_radius: [n_radii][3] (correct, missed, spurious) at radius
 * 0 .. n_radii - 1; n_radii must cover every shift's radius.  planes (float32) and plane_coords: NULL, or room for 16
 * finished examples, oldest first, each [xy labels, xy logits, xz labels, xz logits, yz labels, yz logits] of the crop
 * E (zyx) at z = E0 / 2, y = E1 / 2 and x = E2 / 2 ([E1][E2], [E0][E2], [E0][E1] each), with its stream entry;
 * *n_planes: how many.  reset: then zero the counts and empty the ring (examples in flight are not touched). */
int ffn_examples_tracker(FfnExamples* examples, FfnTrackerCounts* out, int64_t* moves_by_radius, int n_radii,
                         float* planes, FfnExampleCoord* plane_coords, int32_t* n_planes, int reset);
/* n_steps training steps fed by the example loop, with no host copy and one host synchronisation: per step the loop's
 * next batch, ffn_trainer_step's step at learning_rate[i] with unit loss weights, and the logits pasted back.
 * losses_out[i] equals ffn_trainer_step's loss bit for bit.  coords: at least n_steps * batch stream entries;
 * *n_consumed: the entries taken.  Fails for examples of another fov or a batch above the trainer's max_batch. */
int ffn_trainer_train(FfnTrainer* trainer, FfnExamples* examples, const FfnExampleCoord* coords, int64_t n_coords,
                      int n_steps, const float* learning_rate, double* losses_out, int64_t* n_consumed);

/* Known-answer test of the wgmma descriptors (worst absolute error of each case in out[]; see
 * ffn_selftest_wgmma in ffn_b200/csrc/engine.cu).  Used by tests, not by the product path. */
int ffn_selftest_wgmma(int device, double* out, int n_out);

#ifdef __cplusplus
}
#endif
#endif /* FFN_B200_H_ */
