// sb_internal.h — host-side structures shared by the .cu translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "sb_common.cuh"

namespace sb {

// Test hooks: the top twelve bits of the flags word of sb_eval / sb_search_params force a kernel path or a
// search mode that the automatic choice would not take, so that the tests can pin every path and compare the
// forms of the search.  They are not part of the ABI; saturn_b200/_lib.py mirrors the names.
enum : unsigned {
  HOOK_FORCE_GENERIC = 0x80000000u,       // sb_eval: the generic kernel (path 0)
  HOOK_NO_STREAM = 0x40000000u,           // sb_eval: prio rows staged in shared memory, never streamed (tile paths 2 / 1)
  HOOK_NO_FUSED = 0x20000000u,            // search: unfused propose / evaluate / accept rounds
  HOOK_NO_INCREMENTAL = 0x10000000u,      // search: windowed moves, always scored from position 0
  HOOK_VERIFY_INCREMENTAL = 0x08000000u,  // search: also score every incremental proposal from position 0 and count
                                          // the mismatches (sb_search_verify_count)
  HOOK_ROUND1_MOVES = 0x04000000u,        // search: the round-1 move generator (no windows)
  HOOK_PLAIN_ADDR = 0x02000000u,          // sb_eval: plain C++ addressing in the headline tile kernel (ADDR = 0)
  HOOK_WINDOW_BIAS = 0x01000000u,         // search: windows drawn with P(w) ~ w + 1 (experiment, see draw_window)
  HOOK_TABLE_GLOBAL = 0x00800000u,        // position-major scoring: the table in global memory (path 8)
  HOOK_TABLE_PAIR = 0x00400000u,          // position-major scoring: the table split over a CTA pair (path 7)
  HOOK_REORDER = 0x00200000u,             // sb_eval: re-order job-indexed rows into schedule order at any size (path 9)
  HOOK_NO_REORDER = 0x00100000u,          // sb_eval: never re-order job-indexed rows
};
static_assert(((HOOK_FORCE_GENERIC | HOOK_NO_STREAM | HOOK_NO_FUSED | HOOK_NO_INCREMENTAL | HOOK_VERIFY_INCREMENTAL |
                HOOK_ROUND1_MOVES | HOOK_PLAIN_ADDR | HOOK_WINDOW_BIAS | HOOK_TABLE_GLOBAL | HOOK_TABLE_PAIR |
                HOOK_REORDER | HOOK_NO_REORDER) &
               (SB_FLAG_INTEGER_STARTS | SB_FLAG_REDUCED | SB_FLAG_OPT_BY_POSITION | SB_FLAG_POST_KEY |
                SB_FLAG_FOLD_PREV | SB_FLAG_ALT_WARPSCAN | SB_FLAG_SUM_COMPLETION | SB_FLAG_WEIGHTED |
                SB_FLAG_DUE | SB_FLAG_RELEASE | SB_FLAG_MAX_LATENESS | SB_FLAG_LATE_COUNT |
                SB_FLAG_MAX_TARDINESS | SB_FLAG_SQUARED | SB_FLAG_LATE_PENALTY | SB_FLAG_COMPLETION_PENALTY |
                SB_FLAG_WORST_MAKESPAN | SB_FLAG_MEAN_MAKESPAN | SB_FLAG_WORST_TARDINESS | SB_FLAG_MEAN_TARDINESS)) == 0,
              "the test hooks share no bit with the SB_FLAG_* flags");
// The flag space is full up to the hooks: SB_FLAG_MEAN_TARDINESS (0x80000) is the last free bit below HOOK_NO_REORDER.
// A new objective needs a bit freed, or a second word.
static_assert((SB_FLAG_MEAN_TARDINESS << 1) == HOOK_NO_REORDER, "the flags end where the hooks begin");

// Debug options of the streamed tile kernel (sb_debug_tile_options): kept on the handle, not in the flags word, and
// read by sb_eval only.  saturn_b200/_lib.py mirrors the names.
enum TileDebug : unsigned {
  TILE_DEBUG_TIMING = 1u,      // time every tile fetch and the tile loop per warp (sb_debug_tile_wait)
  TILE_DEBUG_ROW_COPIES = 2u,  // one bulk copy per opt row, never one per tile
  TILE_DEBUG_NO_STAGGER = 4u,  // every warp starts at once
};

// Compile-time dispatch: f is called with the run-time value as a type (std::true_type / std::false_type, or the
// prio width as std::integral_constant), so that a launch site names its kernel's template arguments once.
template <class F>
decltype(auto) with_bool(bool b, F&& f) {
  return b ? f(std::true_type{}) : f(std::false_type{});
}
template <class F>
decltype(auto) with_pb(int pb, F&& f) {
  return pb == 1 ? f(std::integral_constant<int, 1>{}) : f(std::integral_constant<int, 2>{});
}
template <Obj O>
using obj_c = std::integral_constant<Obj, O>;
template <class F>
decltype(auto) with_obj(Obj obj, F&& f) {
  switch (obj) {
    case Obj::TailMakespan: return f(obj_c<Obj::TailMakespan>{});
    case Obj::Sum: return f(obj_c<Obj::Sum>{});
    case Obj::WeightedSum: return f(obj_c<Obj::WeightedSum>{});
    case Obj::Tardiness: return f(obj_c<Obj::Tardiness>{});
    case Obj::LateCount: return f(obj_c<Obj::LateCount>{});
    case Obj::MaxTardiness: return f(obj_c<Obj::MaxTardiness>{});
    case Obj::SquaredTardiness: return f(obj_c<Obj::SquaredTardiness>{});
    case Obj::LatePenalty: return f(obj_c<Obj::LatePenalty>{});
    case Obj::CompletionPenalty: return f(obj_c<Obj::CompletionPenalty>{});
    default: return f(obj_c<Obj::Makespan>{});
  }
}
// f(PB, INT, OBJ, R): the prio width, SB_FLAG_INTEGER_STARTS, the objective and SB_FLAG_RELEASE, the template
// arguments that every evaluation and search kernel takes.  R is orthogonal to OBJ: each objective has a release twin.
template <class F>
decltype(auto) with_eval_types(int pb, unsigned flags, Obj obj, F&& f) {
  return with_pb(pb, [&](auto PB) {
    return with_bool(flags & SB_FLAG_INTEGER_STARTS, [&](auto INT) {
      return with_bool(flags & SB_FLAG_RELEASE, [&](auto R) {
        return with_obj(obj, [&](auto OBJ) { return f(PB, INT, OBJ, R); });
      });
    });
  });
}
// The scenario forms run on k_eval_generic, k_eval_full and k_search_pos only, never on the tile kernels: with_obj
// above does not name them, and their launch sites dispatch with this instead.
template <class F>
decltype(auto) with_scenario_types(int pb, unsigned flags, Obj obj, F&& f) {
  return with_pb(pb, [&](auto PB) {
    return with_bool(flags & SB_FLAG_INTEGER_STARTS, [&](auto INT) {
      return with_bool(flags & SB_FLAG_RELEASE, [&](auto R) {
        switch (obj) {
          case Obj::WorstMakespan: return f(PB, INT, obj_c<Obj::WorstMakespan>{}, R);
          case Obj::WorstTardiness: return f(PB, INT, obj_c<Obj::WorstTardiness>{}, R);
          case Obj::MeanTardiness: return f(PB, INT, obj_c<Obj::MeanTardiness>{}, R);
          default: return f(PB, INT, obj_c<Obj::MeanMakespan>{}, R);
        }
      });
    });
  });
}
// the per-job fp32 arrays a kernel stages beside the table: the weights, then the due dates (or tails), then the
// release dates (SB_FLAG_RELEASE), then the late penalties, each where the objective reads it (stage_job_array,
// sb_lane.cuh); each is padded to 16 bytes
inline int job_arrays(Obj obj, unsigned flags) {
  return (obj_weights(obj) ? 1 : 0) + (obj_due(obj) ? 1 : 0) + ((flags & SB_FLAG_RELEASE) ? 1 : 0) +
         (obj_penalty(obj) ? 1 : 0);
}
inline size_t job_array_bytes(int J) { return (static_cast<size_t>(J) * 4 + 15) & ~size_t(15); }

// One kernel launch: raise the kernel's dynamic shared-memory limit to what the launch uses (when it uses any),
// launch, and return the launch error.
template <class... P, class... A>
cudaError_t launch(void (*kern)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, const A&... args) {
  if (smem > 0) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
  }
  kern<<<grid, block, smem, st>>>(args...);
  return cudaGetLastError();
}

struct Device {
  int ordinal = 0;
  int sm_count = 0;
  size_t smem_optin = 0;  // max dynamic shared memory per CTA (227 KB on H100)
};

// peer-memory MIN exchange (sb_xchg.cu)
constexpr int kMaxRanks = 16;
struct XchgDev {
  int rank = 0, world = 1;
  unsigned long long* local = nullptr;            // our mailbox: [2 parities][2] u64 = {key, round}
  unsigned long long* peer[kMaxRanks] = {nullptr};  // every rank's mailbox mapped here (peer[rank] == local)
};
struct XchgPost {
  XchgDev x;
  unsigned long long seq = 0;
  unsigned* counter = nullptr;  // CTA completion counter (zero between launches); null = no fused post
  int fold_prev = 0;            // prologue: fold the peers' keys of round seq-1 into best_key (pipelined exchange)
  int* error = nullptr;         // set to 1 if a peer's round never shows up
};
cudaError_t xchg_post_launch(const XchgDev& x, const unsigned long long* key, unsigned long long seq, cudaStream_t st);
cudaError_t xchg_reduce_launch(const XchgDev& x, unsigned long long seq, unsigned long long* out,
                               unsigned long long* fold, int* error, cudaStream_t st);
cudaError_t xchg_post_reduce_launch(const XchgDev& x, const unsigned long long* key, unsigned long long seq,
                                    unsigned long long* out /*[2]: key, error*/, cudaStream_t st);

struct TilePlan {
  int warps = 0;
  int row_o = 0, row_p = 0, copy_o = 0, copy_p = 0;
  size_t smem = 0;
};

struct EvalCall {
  const float* tab = nullptr;  // canonical table actually used (full or reduced); obj_scenario(obj): the K scaled
                               // copies of it, scenario-major [K][J][SG]
  int K = 0;                   // obj_scenario(obj): the number of scenario tables
  const float* w = nullptr;    // obj_weights(obj): the job weights [J], padded with zeros to a multiple of 4 (unit
                               // weights without SB_FLAG_WEIGHTED)
  const float* d = nullptr;    // obj_due(obj): the job due dates [J] (TailMakespan: the delivery tails max_t d_t - d_j),
                               // padded the same way
  const float* r = nullptr;    // SB_FLAG_RELEASE: the job release dates [J] (ceiled under SB_FLAG_INTEGER_STARTS),
                               // padded the same way
  const float* p = nullptr;    // obj_penalty(obj): the job late penalties [J], padded the same way
  int J = 0, SG = 0;
  const uint8_t* opt = nullptr;
  const uint8_t* prio = nullptr;
  long long B = 0;
  long long stride_o = 0, stride_p = 0;  // bytes
  unsigned flags = 0;
  Obj obj = Obj::Makespan;  // the objective the flags select (decode_objective)
  int nodes = 1;  // > 1: multi-node (reduced table, opt = (node << 3) | (k - 1))
  float* out = nullptr;
  unsigned long long* best_key = nullptr;
  uint32_t id_base = 0;
  int force_generic = 0;
  XchgPost xp;  // fused post of best_key at the end of the tile kernel (tile paths only)
  unsigned tile_debug = 0;                  // the handle's TileDebug options
  unsigned long long* tile_wait = nullptr;  // TILE_DEBUG_TIMING: the handle's two counters (sb_debug_tile_wait)
};

// what the fused search round needs besides an EvalCall (see k_eval_tiles<..., SEARCH = true>)
constexpr int kMaxFusedRounds = 16;
constexpr int kSnapPos = 32;  // schedule positions per window / between state snapshots (incremental search rounds)
struct SearchFuse {
  float* cur_mk = nullptr;        // [chains] makespan of each chain's current candidate
  uint8_t* cur_o = nullptr;       // writable views of the rows the EvalCall reads
  uint8_t* cur_p = nullptr;
  const uint8_t* vopt = nullptr;  // [J][8] proposable opt bytes
  const int* nvalid = nullptr;    // [J]
  uint64_t seed = 0, chain_base = 0;
  int round = 0;    // first round of this launch (RNG counters are keyed by the round number)
  int nrounds = 1;  // rounds run back to back inside one launch, the rows staying on chip (<= kMaxFusedRounds)
  int nodes = 1;
  float temperature[kMaxFusedRounds] = {};  // per round of this launch
  // Tournament resampling inside the tile kernel: before every round r with (r - 1) % resample_every == 0
  // (r > 1) each lane takes over the rows of a random lane of its warp if that lane's candidate is better.
  // `deal` changes which chains share a warp: 0 = chain = tile * 32 + lane, 1 = chain = lane * ntiles + tile.
  int resample_every = 0;
  int deal = 0;
  // Incremental re-evaluation (snap != nullptr; one node only).  Every round a WARP draws one window of
  // kSnapPos schedule positions and its 32 chains make their moves inside that window (windowed moves:
  // `win` = 1), so that all of them can resume the list schedule from the same place: the sorted slot
  // state + running makespan of a chain's CURRENT candidate is snapshotted at every window boundary
  // ([tile][boundary][2 buffers][9 words][32 lanes] floats in HBM/L2, coalesced, valid for one launch), a
  // proposal is scored from the snapshot in front of its window and writes its own boundary states into
  // the other buffer; accepting the move flips which buffer is current (a per-lane bit per boundary), so a
  // rejected move costs nothing to undo.  An unmodified pass at the start of the launch fills the buffers.
  int win = 0;                    // 1: moves are drawn inside a per-warp window (also without snapshots)
  int win_bias = 0;               // 0: windows uniform; 1: P(w) ~ w + 1 (draw_window)
  float* snap = nullptr;          // scratch, (ntiles * nbound * 2 * 9 * 32) floats; nullptr = score every proposal from position 0
  unsigned long long* verify_bad = nullptr;  // test hook: also score from position 0 and count differing results here
  // keep-best in the kernel's tail (KeepBest::counter != nullptr): the CTA that finishes last copies the
  // incumbent's rows when the population's best key improved — saves the separate one-warp launch per round
  struct KeepBest {
    unsigned* counter = nullptr;         // zero between launches
    unsigned long long* keys = nullptr;  // [0] best key of the population, [1] key of the saved encoding
    uint8_t *best_o = nullptr, *best_p = nullptr;
    long long chains = 0, stride_o = 0, stride_p = 0;
  } keep;
};

// arrays: job_arrays(obj, flags), the per-job arrays staged beside the table (unless tab_global: then they all stay in
// global memory)
int plan_tiles(const Device& dev, int J, int SG, int pb, bool stream, int nodes, TilePlan* tp, bool tab_global = false,
               int arrays = 0);
cudaError_t eval_launch(const Device& dev, const EvalCall& c, cudaStream_t st, int* path_used);
cudaError_t eval_alt_launch(const Device& dev, const EvalCall& c, cudaStream_t st);  // sb_eval_alt.cu
int search_round_mode(const Device& dev, int J, int SG, int nodes, int arrays = 0);
cudaError_t search_round_launch(const Device& dev, const EvalCall& c, const SearchFuse& sf, cudaStream_t st);
cudaError_t eval_full_launch(const Device& dev, const EvalCall& c, float* start, uint32_t* slotmask, cudaStream_t st);
// the scenario forms of k_eval_full: the score into c.out and (mks != nullptr) every scenario's makespan, [B][K]
cudaError_t eval_full_scenarios_launch(const Device& dev, const EvalCall& c, float* mks, cudaStream_t st);
cudaError_t validate_launch(const Device& dev, const EvalCall& c, unsigned long long* bad, cudaStream_t st,
                            bool by_pos = false);

// table construction (sb_table.cu); *bad (device) is set to 1 when a cell of T is negative or NaN
cudaError_t build_table_launch(const float* T, int J, int S, int G, uint64_t gcount_packed, float* tab, float* tmin,
                               uint8_t* args, unsigned long long* bad, cudaStream_t st);
// valid (non-dominated, non-sentinel) option lists for the search: vopt[J][8] opt bytes, nvalid[J]
cudaError_t build_valid_launch(const float* tmin, const uint8_t* args, int J, int reduced, float sentinel, uint8_t* vopt,
                               int* nvalid, cudaStream_t st);
// scenario tables: out[k][j][c] = fp32(f[k][j] * tab[j][c]) for the K factor rows f[K][J] (device) and a table of J
// rows of SG cells
cudaError_t scale_tables_launch(const float* tab, int J, int SG, const float* f, int K, float* out, cudaStream_t st);
// shared memory the position-major kernel needs for K scenario tables of J x SG cells beside the per-job arrays the
// objective reads (job_arrays) and the node states; every scenario route is held to it (sb_api.cu: check_per_job)
size_t scenario_smem(int J, int SG, int K, int nodes, unsigned flags, Obj obj);

}  // namespace sb
