// device_types.cuh — plain structs shared by the host engine and the persistent kernel.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ffn_b200.h"

namespace ffn {

constexpr int kThreads = 320;     // warps 0-7: two consumer warpgroups (wgmma + epilogue, 64 accumulator rows each); warp 8: TMA producer;
                                  // warp 9: signals the chains' split-phase barriers (the release stays off the epilogue's path)
constexpr int kLoadWarp = 8;
constexpr int kSigWarp = 9;
#ifndef FFN_ACT_STAGES
#define FFN_ACT_STAGES 3
#endif
constexpr int kActStages = FFN_ACT_STAGES;     // shared-memory ring of per-tile activation operands
constexpr int kTileM = 128;       // accumulator rows per tensor-core tile (two m64 warpgroup MMAs)
constexpr int kTileOut = 126;     // FoV rows a tile OUTPUTS: the dx = -1/+1 partial sums live one row up/down, so
                                  // the first and last accumulator row of every tile only feed their neighbours
constexpr int kStackN = 96;       // MMA N: the three dx taps of a (dz, dy) tap-row stacked along N
constexpr int kFeat = 32;         // feature maps of every hidden layer
constexpr int kAccRegs = 64 * kStackN / 128;   // fp32 accumulators per consumer thread (m64n96 fragment)
constexpr int kMaxConv = 32;      // 2 * depth limit
#ifndef FFN_MAX_CHAINS
#define FFN_MAX_CHAINS 4
#endif
#ifndef FFN_BUFS_PER_CHAIN
#define FFN_BUFS_PER_CHAIN 6
#endif
constexpr int kMaxChains = FFN_MAX_CHAINS;     // flood-fill chains (execution slots) time-multiplexed over the SMs of one kernel
constexpr int kBufsPerChain = FFN_BUFS_PER_CHAIN;  // object buffers per chain: finished objects that wait for their turn to commit are parked
constexpr int kMaxBufs = kMaxChains * kBufsPerChain;
constexpr int kSplitShift = 10;   // FFN_COMPUTE_FP16X2_TC: weights are split as w * 2^10 = hi + lo (keeps lo a normal fp16
                                  // number for |w| down to ~1e-4); the epilogue scales the accumulators back (exact)
constexpr int kMaxTilesPerCta = 0xFFFF / kTileOut;   // the per-CTA step counts are packed into 16 bits (publish_counts)
static_assert(kMaxChains >= 1 && kMaxChains <= 5, "chains");

// Field-of-view geometry in the "row" space the kernels work in.
//
// A FoV voxel (z, y, x) lives at row  r = z * pp + y * xp + x  with xp = fx and pp = (fy + 1) * xp:
// every z-plane is followed by ONE zero line, which supplies the SAME-padding halo of the dy taps
// (dz halos are the zero guard rows before / after the FoV), so a (dz, dy) tap-row is the constant
// row offset dz*pp + dy*xp.  The dx taps need no padding in memory: the tensor-core path stacks them
// along N and adds the neighbouring rows' partial sums in the epilogue (skipping x = 0 / x = fx-1),
// the fp32 path masks them.  Rows are cut into tiles of kTileOut output rows = one 128-row MMA tile.
struct Geom {
  int fz, fy, fx;   // FoV size (z, y, x)
  int mz, my, mx;   // margin = size // 2
  int dz, dy, dx;   // movement deltas
  int nconv;        // number of 3x3x3 convolutions (2 * depth)
  int xp, pp;       // row pitches
  int nr;           // rows spanned by the FoV: (fz-1)*pp + (fy-1)*xp + fx
  int nt;           // tiles: ceil(nr / kTileOut)
  int halo;         // xp + 1: in-plane reach of a tap, in rows
  int guard;        // zero rows before row 0 / after the last tile in global activation buffers
  int rows_alloc;   // guard + nt*128 + guard
  int V;            // fz*fy*fx voxels
  float inv_pp, inv_xp;   // reciprocals for the exact float row decode (checked on the host at engine creation)
};

struct Weights {
  const __half* w16;   // per layer [9 tap-rows][kchunk][12 n-groups][8 n][8 k] fp16 (wgmma K-major, no swizzle),
                       // n = dx * 32 + cout
  const __half* w16x2; // FFN_COMPUTE_FP16X2_TC: per layer the same packing twice, [hi | lo] parts of w * 2^kSplitShift
  const float* w32;    // per layer [27][cin_padded][32] fp32
  const float* bias;   // [nconv][32]
  const float* w_lom;  // [32]
  float b_lom;
};

// Buffers shared by all chains (the fp32 / split-fp16 parity modes run one chain at a time).
constexpr int kTraceEvents = 8, kTraceTiles = 2048, kTraceCta = 1;

struct Workspace {
  __half* act0_l;      // fp16 lo parts (FFN_COMPUTE_FP16X2_TC): x = hi + lo with hi = fp16(x), lo = fp16(x - hi)
  __half* act_l[2];
  float4* act0_f;      // [1][rows_alloc]  (image, seed, 0, 0)
  float4* act_f[2];    // [8][rows_alloc]
  float4* res;         // [8][rows_alloc] fp32 residual stream (fp32 mode)
  unsigned* bar;       // grid barrier counter
  int* abort_flag;     // != 0: a wait timed out, everybody bails
  long long* prof;     // [2][16] cycle counters of CTA 0 and CTA G-1, then [kTraceEvents][kTraceTiles] event times of CTA kTraceCta (profiled build)
};

struct CanvasDev {
  const void* image;
  int image_is_u8;
  float mean, stddev;
  int* seg;
  uint8_t* qprob;             // may be null
  const uint8_t* mask;        // may be null
  const uint8_t* seed_mask;   // may be null
  int sz, sy, sx;
  FfnOptions opt;
  float policy_th_f32;        // smallest float32 >= opt.policy_score_threshold
  int q_cap;                  // capacity of every chain's FIFO
  int traj_cap;               // capacity of every chain's trajectory log
  int* trace;                 // optional event log [cap][4]: (type, z, y, x); null = off
  int trace_cap;
  int lat_dim[3], lat_off[3];
};

// One OBJECT BUFFER: the private state of one object in flight — what the reference keeps in Canvas.seed and the
// FaceMaxMovementPolicy object.  Buffer 0 owns the canvas's own seed array; the others hold objects grown ahead of
// their turn (see Sched).  A chain (execution slot) works on one of its kBufsPerChain buffers at a time.
struct CanvasState;
struct ObjDev {
  float* seed;                // seed canvas of this object (NaN = unvisited)
  float* q_score;             // movement policy FIFO
  int* q_pos;                 // [cap][3]
  unsigned* lattice;          // epoch stamps over the quantised lattice (done set)
  int* traj;                  // [traj_cap][3] FoV positions of the object in flight (speculation check)
  CanvasState* st;
};

// One chain: the step workspace of its FoV.
struct ChainDev {
  __half* act0_h;             // [2][rows_alloc][8] (chunk 1 stays zero)
  __half* act_h[2];           // [4][rows_alloc][8]
  float* seed_raw[2];         // [nt*128] seed FoV as read from the canvas (NaN preserved), by round parity
  float* logits;              // [nt*128] network output (seed + update), before the disco merge
  unsigned* count;            // [2 round parities][2]: voxels with logit >= move threshold; Canvas.history_deleted
  unsigned* bar;              // split-phase barrier of this chain: arrivals of the epilogue groups
  float* res;                 // [nt*128][32] fp32 residual stream of the tensor-core modes, in consumer-thread order (tc_epilogue)
};

enum Phase : int {
  PH_IDLE = 0,
  PH_START_SEGMENT,    // segment_at entry: clear + init (if reset) then pop
  PH_AFTER_CLEAR,
  PH_AFTER_STEP,
  PH_POP,              // resume point inside an object (budget pause)
  PH_NEXT_SEED,
  PH_AFTER_COUNT,
  PH_AFTER_WRITE,
  PH_SEGMENT_DONE,
  PH_ALL_DONE,
  PH_FORCE_STEP,       // update_at: run exactly one step at `cur`
  PH_FINISHED,         // segment_all: the object's flood fill ended; waits for its pastes to land / for its turn to commit
  PH_FREE,             // segment_all: chain has no object (asks the scheduler for a seed every round)
};

// Persistent per-canvas state (global memory) — what the reference keeps in the Canvas and
// FaceMaxMovementPolicy objects between FoV steps.
struct CanvasState {
  int phase;
  int q_head, q_tail;
  unsigned epoch;
  int start[3];
  int cur[3];
  int have_cur;               // cur is the FoV of the step whose logits are in the workspace
  int min_pos[3], max_pos[3];
  long long iters;            // steps of the current object
  int dirty_lo[3], dirty_hi[3];   // box of the seed canvas that may hold non-NaN values (hi exclusive)
  long long seed_index;       // segment_all: index (into the seed list) of the object in flight, -1: restored from a checkpoint
  int spec;                   // segment_all: the object was started ahead of its turn (speculatively)
  int fin_round;              // round in which the object finished (its last paste is visible one round later)
  int reset_seed;             // segment_at: init_seed before starting
  int seg_all;                // 1: segment_all mode, 0: segment_at mode
  int weak;                   // last object ended by 'seed_got_too_weak'
  int popped, pop_run, pop_pos[3];   // leader scratch: queue already popped for this round (phase A)
  int start_max_id;           // Sched::max_id when the object started (scheduler experiments)
  int n_unstepped;            // segment_all: positions that passed Canvas.is_valid_pos but were not stepped on (the pop that ended the
                              // object as 'seed_got_too_weak', pops skipped by the restrictor): logged at the END of the trajectory
                              // buffer, because their verdict — and with it the reference's counters — depends on the labels too
  // commit scratch
  int box_lo[3], box_hi[3];
  unsigned long long cnt_raw, cnt_actual;
  int cur_sid;
  int n_touched;
  unsigned long long seg_t0;  // globaltimer at segment start
  int overflow;               // queue / trajectory capacity exceeded
  int n_trace;                // events written to the trace log
  FfnCounters ctr;            // segment_at / update_at: cumulative; segment_all: counters of the object in flight
};

// Canvas-wide state of segment_all.  The reference processes seeds strictly one after the other
// (inference.py:538-683).  Here up to kMaxChains objects are in flight: the one whose turn it is (`owner`,
// holding seed `commit_idx`) and objects started AHEAD of their turn in private seed arrays.  An object's
// flood fill reads shared state only through `segmentation > 0` tests (inference.py:341,573-581,635), labels
// are only ever added, and every label is written at commit time, in seed order.  So an early run is exactly
// the run the reference would have done iff, when its turn comes, (a) the in-order seed gating still accepts
// the seed and (b) no FoV position it stepped on has been labelled meanwhile; otherwise it is discarded and
// redone in turn.  Results (labels, ids, origins, overlaps, counters) are therefore identical to the
// sequential order, for any number of chains and any choice of early seeds.
struct Sched {
  long long commit_idx;       // seeds [0, commit_idx) are final
  // Every chain has kBufsPerChain object buffers (k * kBufsPerChain ...): `active` is the one it works on, the others
  // are unusable (-1), empty (0), hold a finished object waiting for its turn (1) or a run that was suspended to let
  // such an object commit (2).
  long long bseed[kMaxBufs];          // seed index of the object in a buffer (-1: none)
  int bkind[kMaxBufs];                // -1 unusable, 0 empty, 1 parked, 2 suspended, 3 active
  int bround[kMaxBufs];               // round in which the buffer's object was parked / suspended
  int active[kMaxChains];
  int pad_active;
  int owner;                  // BUFFER holding seed commit_idx (or the restored in-flight object); -1: none
  int nchains;
  int max_id;
  int overflow;               // 1: queue, 2: overlaps, 4: origins, 8: trajectory
  long long n_origins, n_overlaps;
  long long steps_executed;   // FoV steps run, incl. early runs that were discarded
  long long spec_runs, spec_discarded, spec_steps_discarded;
  long long idle_free, idle_wait;   // chain-rounds spent without an object / waiting for the turn to commit
  unsigned round;             // rounds completed (all launches)
  int all_done;
  // Canvas.seed after segment_all holds the LAST object segment_at ran on (inference.py:443-450 clears it only when
  // the next one starts).  `last_chain` is the chain whose seed array holds that object; when that chain is about
  // to start an object ahead of its turn (which may later be discarded), its box is first moved to the snapshot
  // array, so the last in-turn object is never lost.
  int last_chain;             // BUFFER whose seed array holds that object; -1: none
  int last_in_snap;
  int snap_lo[3], snap_hi[3];         // box of the snapshot array holding data (hi exclusive)
  int snap_old_lo[3], snap_old_hi[3]; // previous snapshot box, cleared by the move pass of this round
  FfnCounters ctr;            // committed counters (== the reference's)
};

// Leader -> every CTA, once per round.
struct Ctl {
  int action[kMaxChains];
  int pos[kMaxChains][3];
  int buf[kMaxChains];      // object buffer the chain works on this round
};

enum Mode : int { MODE_PREDICT = 0, MODE_UPDATE_AT = 1, MODE_SEGMENT = 2 };
enum Action : int { ACT_EXIT = 0, ACT_STEP, ACT_CLEAR, ACT_COUNT, ACT_WRITE, ACT_IDLE, ACT_CLEAR_MOVE };

struct Job {
  int mode;
  // predict
  const float* in_seed;
  const float* in_image;
  float* out_logits;
  int batch;
  // update_at
  int pos[3];
  float* pred_out;
  // segment
  long long step_budget;
  const int* seeds;
  long long n_seeds;
  FfnOrigin* origins;
  long long origins_cap;
  FfnOverlap* overlaps;
  long long overlaps_cap;
  int* ovl_count;      // [ovl_ids]
  int* ovl_touched;    // [ovl_ids]
  int ovl_ids;
  unsigned char* seed_status;   // [n_seeds] 0: not started, 1: taken by a chain
  long long round_cap;          // segment_all: rounds one launch may run (watchdog)
  long long watchdog_ns;        // wall-clock limit of one launch
  int debug;                    // scheduler experiments (FFN_B200_DEBUG): 1 = treat every early run as conflicting, 2 = no early runs
};

struct KParams {
  Geom g;
  Weights w;
  Workspace ws;
  CanvasDev cv;
  int nchains;
  ChainDev ch[kMaxChains];
  ObjDev ob[kMaxBufs];
  Sched* sched;
  Ctl* ctl;
  unsigned* round_flag;   // rounds published by the leader (release / acquire)
  // Tensor maps over the fp16 operand buffers of every chain ([0] layer-0 input, [1] / [2] the ping-pong pair):
  // 4-D view (8 halfs, rows, 3 z-planes at pitch pp, k-chunks) so that ONE cp.async.bulk.tensor brings a whole
  // tile's operands — 126 + 2*halo rows of the three z-planes, every k-chunk — into a shared-memory stage.
  CUtensorMap tmap[kMaxChains][3];
  int use_tmap;           // 0: the driver could not encode the maps -> 1-D bulk copies (same shared-memory layout)
  float* snap;            // snapshot seed array (see Sched::last_chain); null with one chain
  Job job;
  int compute_mode;
  int act_smem_bytes;   // 3 * 4 * seg_rows_max * 16
};

// The small-structures area at SmemLayout::bars (byte offsets from there):
//   [0, 160)        mbarriers
//   kOffMisc        s_misc: ints [0, kMaxChains) per-chain step-count accumulators, [7] abort flag copy,
//                   [8, 8 + kMaxChains) disco flags, [16 + 32 k ...) movement-policy scratch of chain k
//   kOffRound       s_round: [2 * kMaxChains][8] ints
//   kOffProf        16 cycle counters (profiled build)
//   kOffXchg        epilogue exchange (4 KB).  The leader's working copies of the chain states
//                   (kStateSlot bytes each) and of the scheduler block ALIAS this region: CTA 0 uses them only between
//                   the grid barrier and the end of leader_round, when no epilogue is running.
constexpr int kStateSlot = 352;
constexpr int kOffMisc = 160;
constexpr int kMiscAbort = 7, kMiscDisco = 8, kMiscScratch = 16;
constexpr int kOffRound = kOffMisc + (kMiscScratch + 32 * kMaxChains) * 4;
constexpr int kOffProf = kOffRound + 2 * kMaxChains * 8 * 4;
constexpr int kOffXchg = (kOffProf + 16 * 8 + 15) / 16 * 16;
constexpr int kXchgBytes = 2 * 8 * 2 * 4 * 8 * 4;   // s_xchg: [2 tile parities][8 warps][2 directions][4 lanes][8]
constexpr int kBarsAreaBytes = kOffXchg + kXchgBytes;

// Shared-memory carve-up (bytes from the 1024-aligned base).
struct SmemLayout {
  int wbuf;        // tc: 2 x 55296 ; fp32: 1 x 110592
  int act;         // tc activation segments
  int bias;        // (nconv + 1) * 32 floats + 4
  int bars;        // mbarriers + scalars
  int total;
};

__host__ __device__ inline SmemLayout smem_layout(const Geom& g) {
  SmemLayout s;
  s.wbuf = 0;
  s.act = 2 * 27 * 4 * 512;   // 110592
  const int seg_rows = kTileOut + 2 * g.halo;               // one tile + halos per stage
  const int act_bytes = kActStages * 3 * 4 * seg_rows * 16;
  s.bias = s.act + act_bytes;
  s.bars = s.bias + (kMaxConv + 1) * 32 * 4 + 16;
  s.total = s.bars + kBarsAreaBytes;
  return s;
}

__host__ __device__ inline size_t w16_layer_offset_halfs(int layer) {
  return layer == 0 ? 0 : (size_t)27 * 2 * 256 + (size_t)(layer - 1) * 27 * 4 * 256;
}
__host__ __device__ inline size_t w32_layer_offset_floats(int layer) {
  return layer == 0 ? 0 : (size_t)27 * 4 * 32 + (size_t)(layer - 1) * 27 * 32 * 32;
}

}  // namespace ffn
