// sb_api.cu — the extern "C" boundary declared in include/saturn_b200.h.
//
// No exceptions cross this boundary and no CPU fallback exists: every entry point either runs
// the CUDA path on the handle's device or returns a negative sb_status with sb_last_error() set.
#include <float.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <new>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "sb_search.h"

using namespace sb;

static thread_local char g_err[512] = "";

static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e__ = (call);                                                                      \
    if (e__ != cudaSuccess)                                                                        \
      return fail(SB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

// The objective a flags word selects (sb_common.cuh: Obj), and whose weights it reads
struct Objective {
  Obj obj = Obj::Makespan;
  bool weighted = false;  // SB_FLAG_WEIGHTED: the caller's weights (sb_set_weights); unit weights otherwise
};

struct SearchState {
  bool ready = false;
  SearchDev d;
  sb_search_params p;
  float scale = 0.f;  // temperature unit: incumbent makespan after initialisation (the sums: sum / J, or weighted
                      // sum / sum of the weights; the due-date objectives: see sb_search_init)
  long long evaluated = 0;
  int rounds_done = 0;
  bool fused_ok = true;  // run rounds with the fused kernel while its tiles fit
  uint8_t *cand_o = nullptr, *cand_p = nullptr;  // device scratch for injected candidates
  unsigned* tail_counter = nullptr;              // keep-best in the fused round's tail (SearchFuse::KeepBest)
  long long launches = 0;                        // fused launches so far (the deal of chains to warps alternates)
  void* blocks[16];
  int nblocks = 0;
  // the allocation is kept across sb_search_init / sb_set_table calls while its shape stays the same (a
  // re-planning loop solves the same task set every interval: no cudaMalloc / cudaFree per solve)
  long long alloc_chains = 0, alloc_stride_o = 0, alloc_stride_p = 0;
  // incremental rounds (tile kernel, one node): boundary snapshots, see SearchFuse::snap
  float* snap = nullptr;
  size_t snap_bytes = 0;
  unsigned long long* verify_bad = nullptr;
  bool win = false, inc = false, verify = false;
  SearchDev alloc;  // the pointers as allocated (s.d's cur / prop pairs trade places when resampling)
  Objective obj;                // the objective of p.flags
  const float* w = nullptr;    // obj_weights: the handle's job weights (or its unit weights)
  const float* due = nullptr;  // obj_due: the handle's due dates (TailMakespan: its delivery tails)
                               // (position-major kernels)
  const float* rel = nullptr;  // SB_FLAG_RELEASE: the handle's release dates as the flags read them (likewise)
  const float* pen = nullptr;  // obj_penalty: the handle's late penalties (likewise)
};

struct sb_handle {
  Device dev;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  int J = 0, S = 0;
  int tab_J = 0, tab_S = 0;  // shape the table buffers are allocated for
  int nodes = 1;
  float sentinel = kSentinel;
  float* tab = nullptr;
  float* tmin = nullptr;
  uint8_t* args = nullptr;
  uint8_t* vopt[2] = {nullptr, nullptr};  // [0] full, [1] reduced
  int* nvalid[2] = {nullptr, nullptr};
  std::vector<float> h_tmin;
  std::vector<uint8_t> h_args;
  unsigned long long* d_scratch = nullptr;  // 4 x u64
  unsigned tile_debug = 0;  // TileDebug options (sb_debug_tile_options)
  unsigned long long* d_tile_wait = nullptr;  // TILE_DEBUG_TIMING: 2 x u64 (sb_debug_tile_wait), allocated on first use
  uint8_t* by_pos = nullptr;  // sb_eval: opt rows re-ordered by schedule position (path 9), grow-only
  size_t by_pos_bytes = 0;
  // staging for sb_eval_host
  cudaStream_t hs[2] = {nullptr, nullptr};
  uint8_t* st_o[2] = {nullptr, nullptr};
  uint8_t* st_p[2] = {nullptr, nullptr};
  float* st_mk[2] = {nullptr, nullptr};
  long long st_cap = 0;
  size_t st_row_o = 0, st_row_p = 0;
  // scratch for decode
  uint8_t* dec_buf = nullptr;
  size_t dec_cap = 0;
  float* stage_T = nullptr;  // device staging of a host table (kept across sb_set_table calls)
  size_t stage_T_bytes = 0;
  // job weights (sb_set_weights): device copy zero-padded to a multiple of 4 floats (16-byte TMA copies), host copy
  // (WSPT seeds) and their sum in double (the temperature unit); has_w is cleared by sb_set_table
  float* d_w = nullptr;
  size_t d_w_cap = 0;
  std::vector<float> h_w;
  double w_sum = 0.0;
  bool has_w = false;
  // SB_FLAG_SQUARED | SB_FLAG_WEIGHTED: whether J * max_j w_j * 2^50 < FLT_MAX (in double), made by sb_set_weights.  A
  // plan inside the 2^24 horizon with |d| < 2^24 has every tardiness below 2^25, so every square below 2^50, and the
  // weighted sum of squares stays finite below that bound; past it the flag is refused
  bool sq_finite = false;
  // due dates (sb_set_due): device copy padded like d_w, J unit weights for SB_FLAG_DUE without SB_FLAG_WEIGHTED,
  // and the host copy (EDD seeds); has_d is cleared by sb_set_table
  float* d_d = nullptr;
  float* d_one = nullptr;
  size_t d_d_cap = 0;
  std::vector<float> h_d;
  bool has_d = false;
  // SB_FLAG_MAX_LATENESS: the delivery tails q_j = max_t d_t - d_j (fp32, padded like d_d; the kernels fold
  // max(C + q) = L_max + max_t d_t >= +0), made by sb_set_due, and whether max d - min d < 2^24 (else even integer
  // due dates give tails that round, and the flag is refused; fractional due dates may round below that too)
  float* d_q = nullptr;
  bool q_exact = false;
  // release dates (sb_set_release): device copies padded like d_w, as given (d_r) and ceiled for
  // SB_FLAG_INTEGER_STARTS (d_rc), and the host copies (seed orders); has_r is cleared by sb_set_table
  float* d_r = nullptr;
  float* d_rc = nullptr;
  size_t d_r_cap = 0;
  std::vector<float> h_r, h_rc;
  bool has_r = false;
  // late penalties (sb_set_penalty): device copy padded like d_w, and their sum in double (the temperature unit);
  // has_p is cleared by sb_set_table
  float* d_p = nullptr;
  size_t d_p_cap = 0;
  double p_sum = 0.0;
  bool has_p = false;
  // runtime scenarios (sb_set_scenarios): the K scaled copies of the full table ([K][J][S][8]) and of the reduced
  // table ([K][J][8]), built on the device from the factors; has_f is cleared by sb_set_table
  float* d_scen = nullptr;
  float* d_scen_min = nullptr;
  float* d_f = nullptr;  // the factors [K][J]
  size_t d_scen_cap = 0, d_scen_min_cap = 0, d_f_cap = 0;
  int scen_K = 0;
  bool has_f = false;
  SearchState search;
  int last_path = -1;
  // peer-memory exchange
  XchgDev xd;
  bool xchg_created = false, xchg_ready = false;
  unsigned long long xseq = 0;
  unsigned* d_xcounter = nullptr;
  int* d_xerr = nullptr;
  void* x_opened[kMaxRanks] = {nullptr};
};

static int use_device(sb_handle* h) {
  if (!h) return fail(SB_ERR_ARG, "null handle");
  CK(cudaSetDevice(h->dev.ordinal));
  return SB_OK;
}

static void free_table(sb_handle* h) {
  cudaFree(h->tab); cudaFree(h->tmin); cudaFree(h->args);
  for (int i = 0; i < 2; ++i) { cudaFree(h->vopt[i]); cudaFree(h->nvalid[i]); h->vopt[i] = nullptr; h->nvalid[i] = nullptr; }
  h->tab = h->tmin = nullptr; h->args = nullptr;
  h->J = h->S = 0;
  h->tab_J = h->tab_S = 0;
}

static void free_search(sb_handle* h) {
  SearchState& s = h->search;
  for (int i = 0; i < s.nblocks; ++i) cudaFree(s.blocks[i]);
  s.nblocks = 0;
  s.ready = false;
  s.d = SearchDev();
  s.alloc = SearchDev();
  s.alloc_chains = s.alloc_stride_o = s.alloc_stride_p = 0;
  s.cand_o = s.cand_p = nullptr;
  s.tail_counter = nullptr;
  s.snap = nullptr;
  s.snap_bytes = 0;
  s.verify_bad = nullptr;
}

static void free_staging(sb_handle* h) {
  for (int i = 0; i < 2; ++i) {
    cudaFree(h->st_o[i]); cudaFree(h->st_p[i]); cudaFree(h->st_mk[i]);
    h->st_o[i] = h->st_p[i] = nullptr; h->st_mk[i] = nullptr;
  }
  h->st_cap = 0;
}

static void free_xchg(sb_handle* h) {
  for (int r = 0; r < kMaxRanks; ++r) {
    if (h->x_opened[r]) cudaIpcCloseMemHandle(h->x_opened[r]);
    h->x_opened[r] = nullptr;
  }
  cudaFree(h->xd.local);
  cudaFree(h->d_xcounter);
  cudaFree(h->d_xerr);
  h->xd = XchgDev();
  h->d_xcounter = nullptr;
  h->d_xerr = nullptr;
  h->xchg_created = h->xchg_ready = false;
  h->xseq = 0;
}

extern "C" {

int sb_abi_version(void) { return SB_ABI_VERSION; }
const char* sb_last_error(void) { return g_err; }

int sb_create(int device, void* stream, sb_handle** out) {
  if (!out) return fail(SB_ERR_ARG, "out is null");
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    return fail(SB_ERR_CUDA, "no CUDA device available (%s); saturn_b200 has no CPU path", cudaGetErrorString(e));
  if (device < 0 || device >= n) return fail(SB_ERR_ARG, "device %d out of range (0..%d)", device, n - 1);
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(SB_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major,
                prop.minor);
  sb_handle* h = new (std::nothrow) sb_handle();
  if (!h) return fail(SB_ERR_NOMEM, "out of host memory");
  h->dev.ordinal = device;
  h->dev.sm_count = prop.multiProcessorCount;
  h->dev.smem_optin = prop.sharedMemPerBlockOptin;
  h->stream = static_cast<cudaStream_t>(stream);  // NULL = the context's default stream
  e = cudaMalloc(&h->d_scratch, 4 * sizeof(unsigned long long));
  if (e != cudaSuccess) { sb_destroy(h); return fail(SB_ERR_CUDA, "cudaMalloc: %s", cudaGetErrorString(e)); }
  for (int i = 0; i < 2; ++i) {
    e = cudaStreamCreateWithFlags(&h->hs[i], cudaStreamNonBlocking);
    if (e != cudaSuccess) { sb_destroy(h); return fail(SB_ERR_CUDA, "cudaStreamCreate: %s", cudaGetErrorString(e)); }
  }
  *out = h;
  return SB_OK;
}

int sb_destroy(sb_handle* h) {
  if (!h) return SB_OK;
  cudaSetDevice(h->dev.ordinal);
  cudaStreamSynchronize(h->stream);
  free_search(h);
  free_table(h);
  free_staging(h);
  free_xchg(h);
  cudaFree(h->d_scratch);
  cudaFree(h->d_tile_wait);
  cudaFree(h->by_pos);
  cudaFree(h->dec_buf);
  cudaFree(h->stage_T);
  cudaFree(h->d_w);
  cudaFree(h->d_f);
  cudaFree(h->d_scen);
  cudaFree(h->d_scen_min);
  cudaFree(h->d_d);
  cudaFree(h->d_one);
  cudaFree(h->d_q);
  cudaFree(h->d_r);
  cudaFree(h->d_rc);
  cudaFree(h->d_p);
  for (int i = 0; i < 2; ++i)
    if (h->hs[i]) cudaStreamDestroy(h->hs[i]);
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return SB_OK;
}

int sb_sync(sb_handle* h) {
  int rc = use_device(h);
  if (rc) return rc;
  CK(cudaStreamSynchronize(h->stream));
  return SB_OK;
}

int sb_set_table(sb_handle* h, const float* T, const uint8_t* gcount, int J, int S, int G, int nodes) {
  int rc = use_device(h);
  if (rc) return rc;
  if (!T || !gcount) return fail(SB_ERR_ARG, "T / gcount is null");
  if (J < 1 || J > 65535) return fail(SB_ERR_ARG, "J=%d outside 1..65535", J);
  if (S < 1 || S > SB_MAX_STRATEGIES) return fail(SB_ERR_ARG, "S=%d outside 1..%d", S, SB_MAX_STRATEGIES);
  if (G < 1 || G > SB_NSLOT) return fail(SB_ERR_ARG, "G=%d outside 1..%d", G, SB_NSLOT);
  if (nodes < 1 || nodes > SB_MAX_NODES) return fail(SB_ERR_ARG, "nodes=%d outside 1..%d", nodes, SB_MAX_NODES);
  uint64_t packed = 0;
  for (int g = 0; g < G; ++g) {
    if (gcount[g] < 1 || gcount[g] > SB_NSLOT) return fail(SB_ERR_ARG, "gcount[%d]=%d outside 1..8", g, gcount[g]);
    packed |= static_cast<uint64_t>(gcount[g]) << (8 * g);
  }
  CK(cudaStreamSynchronize(h->stream));
  h->search.ready = false;  // its buffers are reused by the next sb_search_init if the shape is unchanged
  h->has_w = false;         // weights belong to a task set: a new table needs new ones
  h->has_d = false;         // so do due dates
  h->has_r = false;         // and release dates
  h->has_p = false;         // and late penalties
  h->has_f = false;         // and runtime scenarios
  const size_t nT = static_cast<size_t>(J) * S * G;
  const size_t ntab = static_cast<size_t>(J) * S * kSlots;
  // a re-planning loop sets a table of the same shape every interval: keep the allocations (cudaFree /
  // cudaMalloc synchronise the device and dominate a small solve, above all with one handle per device)
  if (h->tab == nullptr || h->tab_J != J || h->tab_S != S) {
    free_table(h);
    CK(cudaMalloc(&h->tab, ntab * sizeof(float)));
    CK(cudaMalloc(&h->tmin, static_cast<size_t>(J) * kSlots * sizeof(float)));
    CK(cudaMalloc(&h->args, static_cast<size_t>(J) * kSlots));
    for (int i = 0; i < 2; ++i) {
      CK(cudaMalloc(&h->vopt[i], static_cast<size_t>(J) * kSlots));
      CK(cudaMalloc(&h->nvalid[i], static_cast<size_t>(J) * sizeof(int)));
    }
    h->tab_J = J;
    h->tab_S = S;
  }
  h->J = 0;  // not valid until the kernels below have run
  cudaPointerAttributes attr;
  const float* Tdev = T;
  float* tmp = nullptr;
  cudaError_t pe = cudaPointerGetAttributes(&attr, T);
  const bool on_device = (pe == cudaSuccess) && (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged);
  if (pe != cudaSuccess) cudaGetLastError();
  cudaError_t e = cudaSuccess;
  if (!on_device) {
    if (h->stage_T_bytes < nT * sizeof(float)) {
      cudaFree(h->stage_T);
      h->stage_T = nullptr;
      h->stage_T_bytes = 0;
      e = cudaMalloc(&h->stage_T, nT * sizeof(float));
      if (e == cudaSuccess) h->stage_T_bytes = nT * sizeof(float);
    }
    tmp = h->stage_T;
    if (e == cudaSuccess) e = cudaMemcpyAsync(tmp, T, nT * sizeof(float), cudaMemcpyHostToDevice, h->stream);
    Tdev = tmp;
  }
  // d_scratch[0]: set by k_canon_table when a cell is negative or NaN (T may be device memory, so it is checked there)
  unsigned long long bad_cells = 0;
  if (e == cudaSuccess) e = cudaMemsetAsync(h->d_scratch, 0, sizeof(unsigned long long), h->stream);
  if (e == cudaSuccess) e = build_table_launch(Tdev, J, S, G, packed, h->tab, h->tmin, h->args, h->d_scratch, h->stream);
  if (e == cudaSuccess) e = build_valid_launch(h->tmin, h->args, J, 0, h->sentinel, h->vopt[0], h->nvalid[0], h->stream);
  if (e == cudaSuccess) e = build_valid_launch(h->tmin, h->args, J, 1, h->sentinel, h->vopt[1], h->nvalid[1], h->stream);
  h->h_tmin.assign(static_cast<size_t>(J) * kSlots, 0.f);
  h->h_args.assign(static_cast<size_t>(J) * kSlots, 0);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(h->h_tmin.data(), h->tmin, h->h_tmin.size() * sizeof(float), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(h->h_args.data(), h->args, h->h_args.size(), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess)
    e = cudaMemcpyAsync(&bad_cells, h->d_scratch, sizeof(bad_cells), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e != cudaSuccess) {
    free_table(h);
    return fail(SB_ERR_CUDA, "building the table failed: %s", cudaGetErrorString(e));
  }
  if (bad_cells) {
    free_table(h);
    return fail(SB_ERR_ARG, "T holds a negative or NaN runtime (every cell must be >= 0, +inf or a sentinel)");
  }
  h->J = J;
  h->S = S;
  h->nodes = nodes;
  return SB_OK;
}

int sb_set_sentinel(sb_handle* h, float threshold) {
  if (!h) return fail(SB_ERR_ARG, "null handle");
  if (!(threshold > 0.f)) return fail(SB_ERR_ARG, "sentinel threshold must be positive");
  h->sentinel = threshold;
  return SB_OK;
}

int sb_set_weights(sb_handle* h, const float* w, int J) {
  int rc = use_device(h);
  if (rc) return rc;
  if (h->J == 0) return fail(SB_ERR_STATE, "sb_set_table has not been called");
  CK(cudaStreamSynchronize(h->stream));  // no queued kernel may still read the old weights
  h->search.ready = false;               // the running search was set up for the old weights (scale, seeds)
  if (!w) {
    h->has_w = false;
    return SB_OK;
  }
  if (J != h->J) return fail(SB_ERR_ARG, "J=%d differs from the table's J=%d", J, h->J);
  double sum = 0.0, wmax = 0.0;
  for (int j = 0; j < J; ++j) {
    if (!isfinite(w[j]) || !(w[j] > 0.f)) return fail(SB_ERR_ARG, "weight %d (%g) is not finite and > 0", j, w[j]);
    sum += static_cast<double>(w[j]);
    wmax = std::max(wmax, static_cast<double>(w[j]));
  }
  h->sq_finite = static_cast<double>(J) * wmax * 0x1p50 < static_cast<double>(FLT_MAX);
  h->has_w = false;
  const size_t cap = static_cast<size_t>((J + 3) & ~3);
  if (h->d_w_cap < cap) {
    cudaFree(h->d_w);
    h->d_w = nullptr;
    h->d_w_cap = 0;
    CK(cudaMalloc(&h->d_w, cap * sizeof(float)));
    h->d_w_cap = cap;
  }
  h->h_w.assign(w, w + J);
  h->h_w.resize(cap, 0.f);
  CK(cudaMemcpyAsync(h->d_w, h->h_w.data(), cap * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->w_sum = sum;
  h->has_w = true;
  return SB_OK;
}

int sb_set_due(sb_handle* h, const float* d, int J) {
  int rc = use_device(h);
  if (rc) return rc;
  if (h->J == 0) return fail(SB_ERR_STATE, "sb_set_table has not been called");
  CK(cudaStreamSynchronize(h->stream));  // no queued kernel may still read the old due dates
  h->search.ready = false;               // the running search was set up for the old due dates (scale, seeds)
  if (!d) {
    h->has_d = false;
    return SB_OK;
  }
  if (J != h->J) return fail(SB_ERR_ARG, "J=%d differs from the table's J=%d", J, h->J);
  for (int j = 0; j < J; ++j)
    if (!isfinite(d[j]) || !(fabsf(d[j]) < 16777216.f))
      return fail(SB_ERR_ARG, "due date %d (%g) is not finite with |d| < 2^24", j, d[j]);
  h->has_d = false;
  const size_t cap = static_cast<size_t>((J + 3) & ~3);
  if (h->d_d_cap < cap) {
    cudaFree(h->d_d);
    cudaFree(h->d_one);
    cudaFree(h->d_q);
    h->d_d = h->d_one = h->d_q = nullptr;
    h->d_d_cap = 0;
    CK(cudaMalloc(&h->d_d, cap * sizeof(float)));
    CK(cudaMalloc(&h->d_one, cap * sizeof(float)));
    CK(cudaMalloc(&h->d_q, cap * sizeof(float)));
    h->d_d_cap = cap;
  }
  std::vector<float> one(cap, 0.f);
  std::fill(one.begin(), one.begin() + J, 1.f);
  h->h_d.assign(d, d + J);
  h->h_d.resize(cap, 0.f);
  const float dmax = *std::max_element(d, d + J), dmin = *std::min_element(d, d + J);
  h->q_exact = static_cast<double>(dmax) - static_cast<double>(dmin) < 16777216.0;
  // q >= +0: dmax - d is +0 (never -0) where d = dmax
  std::vector<float> q(cap, 0.f);
  for (int j = 0; j < J; ++j) q[j] = dmax - d[j];
  CK(cudaMemcpyAsync(h->d_d, h->h_d.data(), cap * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->d_one, one.data(), cap * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->d_q, q.data(), cap * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->has_d = true;
  return SB_OK;
}

int sb_set_release(sb_handle* h, const float* r, int J) {
  int rc = use_device(h);
  if (rc) return rc;
  if (h->J == 0) return fail(SB_ERR_STATE, "sb_set_table has not been called");
  CK(cudaStreamSynchronize(h->stream));  // no queued kernel may still read the old release dates
  h->search.ready = false;               // the running search was set up for the old release dates (seeds)
  if (!r) {
    h->has_r = false;
    return SB_OK;
  }
  if (J != h->J) return fail(SB_ERR_ARG, "J=%d differs from the table's J=%d", J, h->J);
  for (int j = 0; j < J; ++j)
    if (!isfinite(r[j]) || !(fabsf(r[j]) < 16777216.f))
      return fail(SB_ERR_ARG, "release date %d (%g) is not finite with |r| < 2^24", j, r[j]);
  h->has_r = false;
  const size_t cap = static_cast<size_t>((J + 3) & ~3);
  if (h->d_r_cap < cap) {
    cudaFree(h->d_r);
    cudaFree(h->d_rc);
    h->d_r = h->d_rc = nullptr;
    h->d_r_cap = 0;
    CK(cudaMalloc(&h->d_r, cap * sizeof(float)));
    CK(cudaMalloc(&h->d_rc, cap * sizeof(float)));
    h->d_r_cap = cap;
  }
  // -0 is stored as +0 (x + 0 = x otherwise), so that max(ready, r) with ready = +0 is +0 whatever max does with
  // zeros of both signs: a released job's start keeps its bits
  h->h_r.assign(cap, 0.f);
  for (int j = 0; j < J; ++j) h->h_r[j] = r[j] + 0.f;
  // integer starts: a start >= r is a start >= ceil(r) (exact in fp32 below 2^24), so the step needs no rounding
  h->h_rc.resize(cap);
  for (size_t j = 0; j < cap; ++j) h->h_rc[j] = ceilf(h->h_r[j]) + 0.f;
  CK(cudaMemcpyAsync(h->d_r, h->h_r.data(), cap * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(h->d_rc, h->h_rc.data(), cap * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->has_r = true;
  return SB_OK;
}

int sb_set_penalty(sb_handle* h, const float* p, int J) {
  int rc = use_device(h);
  if (rc) return rc;
  if (h->J == 0) return fail(SB_ERR_STATE, "sb_set_table has not been called");
  CK(cudaStreamSynchronize(h->stream));  // no queued kernel may still read the old penalties
  h->search.ready = false;               // the running search was set up for the old penalties (scale)
  if (!p) {
    h->has_p = false;
    return SB_OK;
  }
  if (J != h->J) return fail(SB_ERR_ARG, "J=%d differs from the table's J=%d", J, h->J);
  double sum = 0.0, pmax = 0.0;
  for (int j = 0; j < J; ++j) {
    if (!isfinite(p[j]) || !(p[j] >= 0.f)) return fail(SB_ERR_ARG, "late penalty %d (%g) is not finite and >= 0", j, p[j]);
    sum += static_cast<double>(p[j]);
    pmax = std::max(pmax, static_cast<double>(p[j]));
  }
  // below J * max p < 2^126 the penalties alone sum below FLT_MAX
  if (!(static_cast<double>(J) * pmax < 0x1p126))
    return fail(SB_ERR_ARG, "J * max p (%g) is not below 2^126: the fp32 sum of the penalties could overflow",
                static_cast<double>(J) * pmax);
  h->has_p = false;
  const size_t cap = static_cast<size_t>((J + 3) & ~3);
  if (h->d_p_cap < cap) {
    cudaFree(h->d_p);
    h->d_p = nullptr;
    h->d_p_cap = 0;
    CK(cudaMalloc(&h->d_p, cap * sizeof(float)));
    h->d_p_cap = cap;
  }
  // -0 is stored as +0 (x + 0 = x otherwise), as sb_set_release stores its release dates
  std::vector<float> hp(cap, 0.f);
  for (int j = 0; j < J; ++j) hp[j] = p[j] + 0.f;
  CK(cudaMemcpyAsync(h->d_p, hp.data(), cap * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->p_sum = sum;
  h->has_p = true;
  return SB_OK;
}

// a device buffer of at least `bytes`, grown (contents dropped) when smaller
static int grow(float** p, size_t* cap, size_t bytes) {
  if (*cap >= bytes) return SB_OK;
  cudaFree(*p);
  *p = nullptr;
  *cap = 0;
  CK(cudaMalloc(p, bytes));
  *cap = bytes;
  return SB_OK;
}

int sb_set_scenarios(sb_handle* h, const float* f, int K, int J) {
  int rc = use_device(h);
  if (rc) return rc;
  if (h->J == 0) return fail(SB_ERR_STATE, "sb_set_table has not been called");
  CK(cudaStreamSynchronize(h->stream));  // no queued kernel may still read the old scenario tables
  h->search.ready = false;               // the running search was set up for the old scenarios
  if (!f) {
    h->has_f = false;
    return SB_OK;
  }
  if (K < 1 || K > 8) return fail(SB_ERR_ARG, "K=%d scenarios outside 1..8", K);
  if (J != h->J) return fail(SB_ERR_ARG, "J=%d differs from the table's J=%d", J, h->J);
  // host or device memory: the factors are checked on the host either way
  const size_t n = static_cast<size_t>(K) * J;
  std::vector<float> hf(n);
  CK(cudaMemcpy(hf.data(), f, n * sizeof(float), cudaMemcpyDefault));
  for (size_t i = 0; i < n; ++i)
    if (!isfinite(hf[i]) || !(hf[i] > 0.f))
      return fail(SB_ERR_ARG, "scenario %d, job %d: factor %g is not finite and > 0", static_cast<int>(i / J),
                  static_cast<int>(i % J), hf[i]);
  h->has_f = false;
  const int SG = h->S * kSlots;
  if ((rc = grow(&h->d_f, &h->d_f_cap, n * sizeof(float)))) return rc;
  if ((rc = grow(&h->d_scen, &h->d_scen_cap, n * SG * sizeof(float)))) return rc;
  if ((rc = grow(&h->d_scen_min, &h->d_scen_min_cap, n * kSlots * sizeof(float)))) return rc;
  CK(cudaMemcpyAsync(h->d_f, hf.data(), n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(scale_tables_launch(h->tab, J, SG, h->d_f, K, h->d_scen, h->stream));
  CK(scale_tables_launch(h->tmin, J, kSlots, h->d_f, K, h->d_scen_min, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->scen_K = K;
  h->has_f = true;
  return SB_OK;
}

// The one reader of the objective flags.  SB_FLAG_WEIGHTED and SB_FLAG_DUE are valid with SB_FLAG_SUM_COMPLETION only;
// SB_FLAG_MAX_LATENESS alone among the objective flags; SB_FLAG_LATE_COUNT, SB_FLAG_MAX_TARDINESS, SB_FLAG_SQUARED,
// SB_FLAG_LATE_PENALTY and SB_FLAG_COMPLETION_PENALTY with SB_FLAG_SUM_COMPLETION | SB_FLAG_DUE only (they change what
// the tardiness form adds per job, and how it folds its terms), and not together or with SB_FLAG_MAX_LATENESS.  Every
// other combination is SB_ERR_ARG.
static int decode_objective(unsigned flags, Objective* o) {
  const bool sum = flags & SB_FLAG_SUM_COMPLETION, weighted = flags & SB_FLAG_WEIGHTED, due = flags & SB_FLAG_DUE;
  const bool lateness = flags & SB_FLAG_MAX_LATENESS, late = flags & SB_FLAG_LATE_COUNT;
  const bool max_tardiness = flags & SB_FLAG_MAX_TARDINESS, squared = flags & SB_FLAG_SQUARED;
  const bool penalty = flags & SB_FLAG_LATE_PENALTY, completion_penalty = flags & SB_FLAG_COMPLETION_PENALTY;
  const bool worst = flags & SB_FLAG_WORST_MAKESPAN, mean = flags & SB_FLAG_MEAN_MAKESPAN;
  const bool worst_t = flags & SB_FLAG_WORST_TARDINESS, mean_t = flags & SB_FLAG_MEAN_TARDINESS;
  if (worst_t && mean_t)
    return fail(SB_ERR_ARG, "SB_FLAG_WORST_TARDINESS and SB_FLAG_MEAN_TARDINESS are two objectives: pass one");
  if ((worst_t || mean_t) && !(sum && due))
    return fail(SB_ERR_ARG, "%s scores the tardiness form over runtime scenarios: it needs SB_FLAG_SUM_COMPLETION and "
                "SB_FLAG_DUE", worst_t ? "SB_FLAG_WORST_TARDINESS" : "SB_FLAG_MEAN_TARDINESS");
  if ((worst_t || mean_t) && (late || max_tardiness || squared || penalty || completion_penalty || lateness || worst ||
                              mean))
    return fail(SB_ERR_ARG, "%s cannot be combined with SB_FLAG_LATE_COUNT, SB_FLAG_MAX_TARDINESS, SB_FLAG_SQUARED, "
                "SB_FLAG_LATE_PENALTY, SB_FLAG_COMPLETION_PENALTY, SB_FLAG_MAX_LATENESS, SB_FLAG_WORST_MAKESPAN or "
                "SB_FLAG_MEAN_MAKESPAN", worst_t ? "SB_FLAG_WORST_TARDINESS" : "SB_FLAG_MEAN_TARDINESS");
  if (worst && mean)
    return fail(SB_ERR_ARG, "SB_FLAG_WORST_MAKESPAN and SB_FLAG_MEAN_MAKESPAN are two objectives: pass one");
  if ((worst || mean) && (sum || weighted || due || lateness || late || max_tardiness || squared || penalty ||
                          completion_penalty))
    return fail(SB_ERR_ARG, "%s scores makespans over runtime scenarios: it cannot be combined with "
                "SB_FLAG_SUM_COMPLETION, SB_FLAG_WEIGHTED, SB_FLAG_DUE, SB_FLAG_MAX_LATENESS, SB_FLAG_LATE_COUNT, "
                "SB_FLAG_MAX_TARDINESS, SB_FLAG_SQUARED, SB_FLAG_LATE_PENALTY or SB_FLAG_COMPLETION_PENALTY",
                worst ? "SB_FLAG_WORST_MAKESPAN" : "SB_FLAG_MEAN_MAKESPAN");
  if (completion_penalty && !(sum && due))
    return fail(SB_ERR_ARG, "SB_FLAG_COMPLETION_PENALTY adds a fixed penalty per missed due date to the completion "
                "time: it needs SB_FLAG_SUM_COMPLETION and SB_FLAG_DUE");
  if (completion_penalty && (penalty || late || max_tardiness || squared || lateness))
    return fail(SB_ERR_ARG, "SB_FLAG_COMPLETION_PENALTY cannot be combined with SB_FLAG_LATE_PENALTY, "
                "SB_FLAG_LATE_COUNT, SB_FLAG_MAX_TARDINESS, SB_FLAG_SQUARED or SB_FLAG_MAX_LATENESS");
  if (penalty && !(sum && due))
    return fail(SB_ERR_ARG, "SB_FLAG_LATE_PENALTY adds a fixed penalty to the tardiness form's late terms: it needs "
                "SB_FLAG_SUM_COMPLETION and SB_FLAG_DUE");
  if (penalty && (late || max_tardiness || squared || lateness))
    return fail(SB_ERR_ARG, "SB_FLAG_LATE_PENALTY cannot be combined with SB_FLAG_LATE_COUNT, SB_FLAG_MAX_TARDINESS, "
                "SB_FLAG_SQUARED or SB_FLAG_MAX_LATENESS");
  if (squared && !(sum && due))
    return fail(SB_ERR_ARG, "SB_FLAG_SQUARED squares the tardiness form's terms: it needs SB_FLAG_SUM_COMPLETION and "
                "SB_FLAG_DUE");
  if (squared && (late || max_tardiness || lateness))
    return fail(SB_ERR_ARG, "SB_FLAG_SQUARED cannot be combined with SB_FLAG_LATE_COUNT, SB_FLAG_MAX_TARDINESS or "
                "SB_FLAG_MAX_LATENESS");
  if (late && !(sum && due))
    return fail(SB_ERR_ARG, "SB_FLAG_LATE_COUNT counts late jobs on the tardiness form: it needs SB_FLAG_SUM_COMPLETION "
                "and SB_FLAG_DUE");
  if (max_tardiness && !(sum && due))
    return fail(SB_ERR_ARG, "SB_FLAG_MAX_TARDINESS folds the tardiness form with max: it needs SB_FLAG_SUM_COMPLETION "
                "and SB_FLAG_DUE");
  if (max_tardiness && (late || lateness))
    return fail(SB_ERR_ARG, "SB_FLAG_MAX_TARDINESS cannot be combined with SB_FLAG_LATE_COUNT or SB_FLAG_MAX_LATENESS");
  if (lateness && (sum || weighted || due))
    return fail(SB_ERR_ARG, "SB_FLAG_MAX_LATENESS is an objective of its own: it cannot be combined with "
                "SB_FLAG_SUM_COMPLETION, SB_FLAG_WEIGHTED or SB_FLAG_DUE");
  if (weighted && !sum)
    return fail(SB_ERR_ARG, "SB_FLAG_WEIGHTED weights the sum of completion times: it needs SB_FLAG_SUM_COMPLETION");
  if (due && !sum)
    return fail(SB_ERR_ARG, "SB_FLAG_DUE scores the tardiness of the completion times: it needs SB_FLAG_SUM_COMPLETION");
  o->weighted = weighted;
  if (worst) o->obj = Obj::WorstMakespan;
  else if (mean) o->obj = Obj::MeanMakespan;
  else if (lateness) o->obj = Obj::TailMakespan;
  else if (!sum) o->obj = Obj::Makespan;
  else if (late) o->obj = Obj::LateCount;
  else if (max_tardiness) o->obj = Obj::MaxTardiness;
  else if (squared) o->obj = Obj::SquaredTardiness;
  else if (penalty) o->obj = Obj::LatePenalty;
  else if (completion_penalty) o->obj = Obj::CompletionPenalty;
  else if (worst_t) o->obj = Obj::WorstTardiness;
  else if (mean_t) o->obj = Obj::MeanTardiness;
  else if (due) o->obj = Obj::Tardiness;
  else o->obj = weighted ? Obj::WeightedSum : Obj::Sum;
  return SB_OK;
}

// the objectives folded from the tardiness form (SB_FLAG_DUE): their scores reach +0, which no plan can beat (run with
// every due date +0, as the worst and mean completion time, the scenario forms never do with a nonzero runtime)
static bool tardiness_form(Obj o) {
  return o == Obj::Tardiness || o == Obj::LateCount || o == Obj::MaxTardiness || o == Obj::SquaredTardiness ||
         o == Obj::LatePenalty || o == Obj::WorstTardiness || o == Obj::MeanTardiness;
}
// the flag that names a scenario form, for messages
static const char* scenario_flag_name(Obj o) {
  switch (o) {
    case Obj::WorstMakespan: return "SB_FLAG_WORST_MAKESPAN";
    case Obj::MeanMakespan: return "SB_FLAG_MEAN_MAKESPAN";
    case Obj::WorstTardiness: return "SB_FLAG_WORST_TARDINESS";
    default: return "SB_FLAG_MEAN_TARDINESS";
  }
}

// decode_objective, then the per-job arrays the objective reads (and SB_FLAG_RELEASE's) must be set on the handle
static int check_per_job(const sb_handle* h, unsigned flags, Objective* o) {
  if (int rc = decode_objective(flags, o)) return rc;
  if (o->obj == Obj::TailMakespan) {
    if (!h->has_d) return fail(SB_ERR_STATE, "SB_FLAG_MAX_LATENESS needs sb_set_due (sb_set_table clears the due dates)");
    if (!h->q_exact)
      return fail(SB_ERR_ARG, "SB_FLAG_MAX_LATENESS needs max d - min d < 2^24 (beyond it the tails max d - d round even "
                  "for integer due dates)");
  }
  if (o->weighted && !h->has_w)
    return fail(SB_ERR_STATE, "SB_FLAG_WEIGHTED needs sb_set_weights (sb_set_table clears the weights)");
  if (obj_due(o->obj) && !h->has_d)
    return fail(SB_ERR_STATE, "SB_FLAG_DUE needs sb_set_due (sb_set_table clears the due dates)");
  if (o->obj == Obj::SquaredTardiness && o->weighted && !h->sq_finite)
    return fail(SB_ERR_ARG, "SB_FLAG_SQUARED | SB_FLAG_WEIGHTED needs J * max w * 2^50 < FLT_MAX (beyond it the sum of "
                "squared tardiness can overflow fp32)");
  if (obj_penalty(o->obj) && !h->has_p)
    return fail(SB_ERR_STATE, "%s needs sb_set_penalty (sb_set_table clears the penalties)",
                o->obj == Obj::CompletionPenalty ? "SB_FLAG_COMPLETION_PENALTY" : "SB_FLAG_LATE_PENALTY");
  if ((flags & SB_FLAG_RELEASE) && !h->has_r)
    return fail(SB_ERR_STATE, "SB_FLAG_RELEASE needs sb_set_release (sb_set_table clears the release dates)");
  if (obj_scenario(o->obj)) {
    const char* name = scenario_flag_name(o->obj);
    if (!h->has_f) return fail(SB_ERR_STATE, "%s needs sb_set_scenarios (sb_set_table clears the scenarios)", name);
    if (flags & SB_FLAG_ALT_WARPSCAN)
      return fail(SB_ERR_UNSUPPORTED, "%s is not available with SB_FLAG_ALT_WARPSCAN", name);
    const int SG = ((flags & SB_FLAG_REDUCED) ? 1 : h->S) * kSlots;
    const size_t need = scenario_smem(h->J, SG, h->scen_K, h->nodes, flags, o->obj);
    if (need > h->dev.smem_optin)
      return fail(SB_ERR_UNSUPPORTED, "%s: the %d scenario tables of %d x %d cells (%zu bytes with the per-job arrays "
                  "and node states) must fit in one CTA's shared memory (%zu bytes); pass SB_FLAG_REDUCED or fewer "
                  "scenarios", name, h->scen_K, h->J, SG, need, h->dev.smem_optin);
  }
  return SB_OK;
}
// the release dates the kernels read: ceiled under SB_FLAG_INTEGER_STARTS, as given otherwise, or none
static const float* job_release(const sb_handle* h, unsigned flags) {
  if (!(flags & SB_FLAG_RELEASE)) return nullptr;
  return (flags & SB_FLAG_INTEGER_STARTS) ? h->d_rc : h->d_r;
}
// the due-date array the kernels read: the due dates, TailMakespan's delivery tails, or none
static const float* job_due(const sb_handle* h, Obj obj) {
  if (!obj_due(obj)) return nullptr;
  return obj == Obj::TailMakespan ? h->d_q : h->d_d;
}
// the late penalties the kernels read, or none
static const float* job_penalty(const sb_handle* h, Obj obj) { return obj_penalty(obj) ? h->d_p : nullptr; }
// the weights the kernels read: the caller's, unit weights, or none
static const float* job_weights(const sb_handle* h, const Objective& o) {
  if (!obj_weights(o.obj)) return nullptr;
  return o.weighted ? h->d_w : h->d_one;
}

int sb_get_reduced(sb_handle* h, float* tmin, uint8_t* args) {
  if (!h) return fail(SB_ERR_ARG, "null handle");
  if (h->J == 0) return fail(SB_ERR_STATE, "sb_set_table has not been called");
  if (tmin) memcpy(tmin, h->h_tmin.data(), h->h_tmin.size() * sizeof(float));
  if (args) memcpy(args, h->h_args.data(), h->h_args.size());
  return SB_OK;
}

static int make_call(sb_handle* h, const uint8_t* opt, const void* prio, int64_t B, int64_t row_stride, unsigned flags,
                     EvalCall* c, bool by_position_ok = false) {
  if (h->J == 0) return fail(SB_ERR_STATE, "sb_set_table has not been called");
  if ((flags & SB_FLAG_OPT_BY_POSITION) && !by_position_ok)
    return fail(SB_ERR_UNSUPPORTED, "SB_FLAG_OPT_BY_POSITION is accepted by sb_eval only");
  if (B < 0) return fail(SB_ERR_ARG, "B=%lld is negative", static_cast<long long>(B));
  if (B > 0 && (!opt || !prio)) return fail(SB_ERR_ARG, "opt / prio is null");
  if (row_stride < h->J) return fail(SB_ERR_ARG, "row_stride=%lld < J=%d", static_cast<long long>(row_stride), h->J);
  Objective o;
  if (int rc = check_per_job(h, flags, &o)) return rc;
  if (B > 0xffffffffll) return fail(SB_ERR_ARG, "B=%lld exceeds 2^32-1 candidates per call", static_cast<long long>(B));
  const int pb = h->J <= 256 ? 1 : 2;
  const bool reduced = (flags & SB_FLAG_REDUCED) != 0;
  if (h->nodes > 1 && !reduced)
    return fail(SB_ERR_UNSUPPORTED, "a %d-node table is evaluated on the reduced table only: pass SB_FLAG_REDUCED "
                "(opt byte = (node << 3) | (k - 1))", h->nodes);
  c->nodes = h->nodes;
  c->tab = reduced ? h->tmin : h->tab;
  if (obj_scenario(o.obj)) {
    c->tab = reduced ? h->d_scen_min : h->d_scen;
    c->K = h->scen_K;
  }
  c->J = h->J;
  c->SG = (reduced ? 1 : h->S) * kSlots;
  c->opt = opt;
  c->prio = static_cast<const uint8_t*>(prio);
  c->B = B;
  c->stride_o = row_stride;
  c->stride_p = row_stride * pb;
  c->flags = flags;
  c->obj = o.obj;
  c->w = job_weights(h, o);
  c->d = job_due(h, o.obj);
  c->r = job_release(h, flags);
  c->p = job_penalty(h, o.obj);
  return SB_OK;
}

int sb_eval(sb_handle* h, const uint8_t* opt, const void* prio, int64_t B, int64_t row_stride, unsigned flags,
            float* makespan_out, uint64_t* best_key, uint32_t id_base) {
  int rc = use_device(h);
  if (rc) return rc;
  EvalCall c;
  rc = make_call(h, opt, prio, B, row_stride, flags, &c, true);
  if (rc) return rc;
  if (B > 0 && !makespan_out) return fail(SB_ERR_ARG, "makespan_out is null");
  c.out = makespan_out;
  c.best_key = reinterpret_cast<unsigned long long*>(best_key);
  c.id_base = id_base;
  if (flags & SB_FLAG_OPT_BY_POSITION) {
    if (flags & (SB_FLAG_POST_KEY | SB_FLAG_FOLD_PREV))
      return fail(SB_ERR_UNSUPPORTED, "SB_FLAG_OPT_BY_POSITION cannot be combined with the fused key exchange");
    int path = 5;
    cudaError_t e = eval_pos_launch(h->dev, c, h->stream, &path);
    if (e == cudaErrorNotSupported) {
      cudaGetLastError();
      return fail(SB_ERR_UNSUPPORTED, "SB_FLAG_OPT_BY_POSITION needs 32-byte aligned rows (row_stride %% 32 == 0) and a "
                  "multi-node table that fits in shared memory (J*32 bytes <= %zu)", h->dev.smem_optin - 16);
    }
    CK(e);
    h->last_path = path;
    return SB_OK;
  }
  // Job-indexed rows where the tile kernel runs short of shared memory — a table that does not fit beside the
  // tiles (C5 with all strategies: 256 KB, tile kernel path 4) or J >= 1024 (33 KB of opt tile per warp: 5 warps
  // per SM): re-order the opt bytes into schedule order on the device (h->by_pos, B x row_stride bytes, grow-only)
  // and score them with the position-major kernel, which keeps no tile and streams both rows.
  // HOOK_REORDER takes this route at any size.
  {
    // the scenario forms take this route under HOOK_REORDER only: their tables fit the generic kernel's shared memory
    const bool hooks = (flags & (HOOK_FORCE_GENERIC | HOOK_NO_STREAM | HOOK_NO_REORDER | SB_FLAG_POST_KEY |
                                 SB_FLAG_FOLD_PREV | SB_FLAG_ALT_WARPSCAN)) != 0 ||
                       (obj_scenario(c.obj) && !(flags & HOOK_REORDER));
    const bool aligned = row_stride % 32 == 0 && reinterpret_cast<uintptr_t>(opt) % 32 == 0 &&
                         reinterpret_cast<uintptr_t>(prio) % 32 == 0;
    const int home = eval_pos_home(h->dev, c.J, c.SG, c.nodes, flags, c.obj, c.K);
    if (!hooks && aligned && B > 0 && c.J <= 6144 && home >= 0 && (home != 0 || c.J >= 1024 || (flags & HOOK_REORDER))) {
      const size_t need = static_cast<size_t>(B) * static_cast<size_t>(row_stride);
      if (need > h->by_pos_bytes) {
        if (h->by_pos) CK(cudaFree(h->by_pos));
        h->by_pos = nullptr;
        h->by_pos_bytes = 0;
        CK(cudaMalloc(&h->by_pos, need));
        h->by_pos_bytes = need;
      }
      CK(opt_by_position_launch(h->dev, c, h->by_pos, h->stream));
      EvalCall cp = c;
      cp.opt = h->by_pos;
      int path = 5;
      CK(eval_pos_launch(h->dev, cp, h->stream, &path));
      h->last_path = 9;
      return SB_OK;
    }
  }
  if (flags & SB_FLAG_ALT_WARPSCAN) {
    if (c.obj != Obj::Makespan || (flags & SB_FLAG_RELEASE))
      return fail(SB_ERR_UNSUPPORTED, "SB_FLAG_ALT_WARPSCAN scores the makespan without release dates only: it "
                  "cannot be combined with SB_FLAG_SUM_COMPLETION, SB_FLAG_WEIGHTED, SB_FLAG_DUE, SB_FLAG_RELEASE, "
                  "SB_FLAG_MAX_LATENESS, SB_FLAG_LATE_COUNT, SB_FLAG_MAX_TARDINESS, SB_FLAG_SQUARED, "
                  "SB_FLAG_LATE_PENALTY or SB_FLAG_COMPLETION_PENALTY");
    if (flags & (SB_FLAG_POST_KEY | SB_FLAG_FOLD_PREV))
      return fail(SB_ERR_UNSUPPORTED, "SB_FLAG_ALT_WARPSCAN cannot be combined with the fused key exchange");
    cudaError_t e = eval_alt_launch(h->dev, c, h->stream);
    if (e == cudaErrorNotSupported) {
      cudaGetLastError();
      return fail(SB_ERR_UNSUPPORTED, "SB_FLAG_ALT_WARPSCAN needs one node and a table that fits in shared memory");
    }
    CK(e);
    h->last_path = 6;
    return SB_OK;
  }
  c.force_generic = (flags & HOOK_FORCE_GENERIC) ? 1 : 0;
  c.tile_debug = h->tile_debug;
  if (h->tile_debug & TILE_DEBUG_TIMING) {
    if (!h->d_tile_wait) {
      CK(cudaMalloc(&h->d_tile_wait, 2 * sizeof(unsigned long long)));
      CK(cudaMemsetAsync(h->d_tile_wait, 0, 2 * sizeof(unsigned long long), h->stream));
    }
    c.tile_wait = h->d_tile_wait;
  }
  const bool post = (flags & SB_FLAG_POST_KEY) != 0;
  if (post) {
    if (!h->xchg_ready) return fail(SB_ERR_STATE, "SB_FLAG_POST_KEY needs sb_xchg_connect first");
    if (!best_key) return fail(SB_ERR_ARG, "SB_FLAG_POST_KEY needs best_key");
    c.xp.x = h->xd;
    c.xp.seq = ++h->xseq;
    c.xp.counter = h->d_xcounter;
    c.xp.fold_prev = (flags & SB_FLAG_FOLD_PREV) ? 1 : 0;
    c.xp.error = h->d_xerr;
  }
  CK(eval_launch(h->dev, c, h->stream, &h->last_path));
  if (post && (h->last_path == 0 || B == 0)) {
    // the generic kernel has neither the fused prologue nor the fused tail: do both with the small kernels
    if (c.xp.fold_prev && h->xseq > 1)
      CK(xchg_reduce_launch(h->xd, h->xseq - 1, h->d_scratch + 1, reinterpret_cast<unsigned long long*>(best_key),
                            h->d_xerr, h->stream));
    CK(xchg_post_launch(h->xd, reinterpret_cast<unsigned long long*>(best_key), h->xseq, h->stream));
  }
  return SB_OK;
}

int sb_last_eval_path(sb_handle* h) { return h ? h->last_path : -1; }

int sb_validate(sb_handle* h, const uint8_t* opt, const void* prio, int64_t B, int64_t row_stride, unsigned flags,
                int64_t* bad_rows) {
  int rc = use_device(h);
  if (rc) return rc;
  EvalCall c;
  rc = make_call(h, opt, prio, B, row_stride, flags, &c);
  if (rc) return rc;
  if (!bad_rows) return fail(SB_ERR_ARG, "bad_rows is null");
  c.tab = (flags & SB_FLAG_REDUCED) ? h->tmin : h->tab;  // the cells a candidate selects exist in the nominal table
  CK(cudaMemsetAsync(h->d_scratch, 0, sizeof(unsigned long long), h->stream));
  CK(validate_launch(h->dev, c, h->d_scratch, h->stream));
  unsigned long long bad = 0;
  CK(cudaMemcpyAsync(&bad, h->d_scratch, sizeof(bad), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  *bad_rows = static_cast<int64_t>(bad);
  return SB_OK;
}

// The slot-exact kernel under any objective.  The scenario forms score on their tables, and their start times and slot
// masks are those of the nominal schedule: the makespan form on the nominal table writes them.
static cudaError_t eval_full_any(sb_handle* h, const EvalCall& c, float* start, uint32_t* slotmask, float* mks) {
  if (!obj_scenario(c.obj)) return eval_full_launch(h->dev, c, start, slotmask, h->stream);
  if (start || slotmask) {
    EvalCall nominal = c;
    nominal.obj = Obj::Makespan;
    nominal.K = 0;
    nominal.tab = (c.flags & SB_FLAG_REDUCED) ? h->tmin : h->tab;
    nominal.out = nullptr;
    cudaError_t e = eval_full_launch(h->dev, nominal, start, slotmask, h->stream);
    if (e != cudaSuccess) return e;
  }
  return eval_full_scenarios_launch(h->dev, c, mks, h->stream);
}

int sb_eval_full(sb_handle* h, const uint8_t* opt, const void* prio, int64_t B, int64_t row_stride, unsigned flags,
                 float* makespan_out, float* start_out, uint32_t* slotmask_out) {
  int rc = use_device(h);
  if (rc) return rc;
  EvalCall c;
  rc = make_call(h, opt, prio, B, row_stride, flags, &c);
  if (rc) return rc;
  c.out = makespan_out;
  CK(eval_full_any(h, c, start_out, slotmask_out, nullptr));
  return SB_OK;
}

int sb_eval_scenarios(sb_handle* h, const uint8_t* opt, const void* prio, int64_t B, int64_t row_stride, unsigned flags,
                      float* score_out, float* makespans_out) {
  int rc = use_device(h);
  if (rc) return rc;
  EvalCall c;
  rc = make_call(h, opt, prio, B, row_stride, flags, &c);
  if (rc) return rc;
  if (!obj_scenario(c.obj))
    return fail(SB_ERR_ARG, "sb_eval_scenarios needs SB_FLAG_WORST_MAKESPAN, SB_FLAG_MEAN_MAKESPAN, "
                "SB_FLAG_WORST_TARDINESS or SB_FLAG_MEAN_TARDINESS");
  if (B > 0 && !makespans_out) return fail(SB_ERR_ARG, "makespans_out is null");
  c.out = score_out;
  CK(eval_full_scenarios_launch(h->dev, c, makespans_out, h->stream));
  return SB_OK;
}

static int ensure_staging(sb_handle* h, long long cap, size_t row_o, size_t row_p) {
  if (h->st_cap >= cap && h->st_row_o == row_o && h->st_row_p == row_p) return SB_OK;
  free_staging(h);
  for (int i = 0; i < 2; ++i) {
    CK(cudaMalloc(&h->st_o[i], static_cast<size_t>(cap) * row_o));
    CK(cudaMalloc(&h->st_p[i], static_cast<size_t>(cap) * row_p));
    CK(cudaMalloc(&h->st_mk[i], static_cast<size_t>(cap) * sizeof(float)));
  }
  h->st_cap = cap;
  h->st_row_o = row_o;
  h->st_row_p = row_p;
  return SB_OK;
}

int sb_eval_host(sb_handle* h, const uint8_t* opt, const void* prio, int64_t B, int64_t row_stride, unsigned flags,
                 float* makespan_out) {
  int rc = use_device(h);
  if (rc) return rc;
  EvalCall c;
  rc = make_call(h, opt, prio, B, row_stride, flags, &c);
  if (rc) return rc;
  if (B == 0) return SB_OK;
  if (!makespan_out) return fail(SB_ERR_ARG, "makespan_out is null");
  // chunk = a few full waves of 32-candidate tiles over all SMs, so copies overlap kernels
  const long long wave = static_cast<long long>(h->dev.sm_count) * 8 * 32;
  long long chunk = wave * 4;
  if (chunk > B) chunk = B;
  rc = ensure_staging(h, chunk, static_cast<size_t>(c.stride_o), static_cast<size_t>(c.stride_p));
  if (rc) return rc;
  CK(cudaStreamSynchronize(h->stream));
  const uint8_t* ho = opt;
  const uint8_t* hp = static_cast<const uint8_t*>(prio);
  int slot = 0;
  for (long long b0 = 0; b0 < B; b0 += chunk, slot ^= 1) {
    const long long nb = (B - b0 < chunk) ? (B - b0) : chunk;
    cudaStream_t st = h->hs[slot];
    CK(cudaMemcpyAsync(h->st_o[slot], ho + b0 * c.stride_o, static_cast<size_t>(nb) * c.stride_o, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(h->st_p[slot], hp + b0 * c.stride_p, static_cast<size_t>(nb) * c.stride_p, cudaMemcpyHostToDevice, st));
    EvalCall cc = c;
    cc.opt = h->st_o[slot];
    cc.prio = h->st_p[slot];
    cc.B = nb;
    cc.out = h->st_mk[slot];
    CK(eval_launch(h->dev, cc, st, &h->last_path));
    CK(cudaMemcpyAsync(makespan_out + b0, h->st_mk[slot], static_cast<size_t>(nb) * sizeof(float), cudaMemcpyDeviceToHost, st));
  }
  CK(cudaStreamSynchronize(h->hs[0]));
  CK(cudaStreamSynchronize(h->hs[1]));
  return SB_OK;
}

int sb_decode(sb_handle* h, const uint8_t* opt, const void* prio, unsigned flags, float* start, uint32_t* slotmask,
              uint8_t* strategy, uint8_t* gpus, uint8_t* node, float* makespan) {
  int rc = use_device(h);
  if (rc) return rc;
  if (h->J == 0) return fail(SB_ERR_STATE, "sb_set_table has not been called");
  if (!opt || !prio) return fail(SB_ERR_ARG, "opt / prio is null");
  const int J = h->J;
  const int pb = J <= 256 ? 1 : 2;
  const size_t need = static_cast<size_t>(J) * (1 + pb) + static_cast<size_t>(J) * 8 + 16 + 64;
  if (h->dec_cap < need) {
    cudaFree(h->dec_buf);
    h->dec_buf = nullptr;
    h->dec_cap = 0;
    CK(cudaMalloc(&h->dec_buf, need));
    h->dec_cap = need;
  }
  // layout: [start f32 J][mask u32 J][mk f32 (16B)][opt J][prio J*pb]
  float* d_start = reinterpret_cast<float*>(h->dec_buf);
  uint32_t* d_mask = reinterpret_cast<uint32_t*>(h->dec_buf + static_cast<size_t>(J) * 4);
  float* d_mk = reinterpret_cast<float*>(h->dec_buf + static_cast<size_t>(J) * 8);
  uint8_t* d_opt = h->dec_buf + static_cast<size_t>(J) * 8 + 16;
  uint8_t* d_prio = d_opt + ((J + 1) & ~1);
  CK(cudaMemcpyAsync(d_opt, opt, J, cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(d_prio, prio, static_cast<size_t>(J) * pb, cudaMemcpyHostToDevice, h->stream));
  EvalCall c;
  rc = make_call(h, d_opt, d_prio, 1, J, flags, &c);
  if (rc) return rc;
  c.out = d_mk;
  CK(eval_full_any(h, c, d_start, d_mask, nullptr));
  std::vector<float> hs(J);
  std::vector<uint32_t> hm(J);
  float mk = 0.f;
  CK(cudaMemcpyAsync(hs.data(), d_start, static_cast<size_t>(J) * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(hm.data(), d_mask, static_cast<size_t>(J) * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaMemcpyAsync(&mk, d_mk, 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  const bool reduced = (flags & SB_FLAG_REDUCED) != 0;
  for (int j = 0; j < J; ++j) {
    if (start) start[j] = hs[j];
    if (slotmask) slotmask[j] = hm[j] & 0xffffu;
    if (node) node[j] = static_cast<uint8_t>(hm[j] >> 16);
    const int col = opt[j] & 7;
    if (gpus) gpus[j] = static_cast<uint8_t>(col + 1);
    if (strategy)
      strategy[j] = reduced ? h->h_args[static_cast<size_t>(j) * kSlots + col] : static_cast<uint8_t>(opt[j] >> 3);
  }
  if (makespan) *makespan = mk;
  return SB_OK;
}

// ------------------------------------------------------------------------------------------ exchange
// a fresh, zeroed mailbox, completion counter and error flag on the handle's device, for rank `rank` of `world`
static int create_mailbox(sb_handle* h, int rank, int world) {
  free_xchg(h);
  const size_t bytes = 2 * kMaxRanks * 2 * sizeof(unsigned long long);
  CK(cudaMalloc(&h->xd.local, bytes));
  CK(cudaMemset(h->xd.local, 0, bytes));
  CK(cudaMalloc(&h->d_xcounter, sizeof(unsigned)));
  CK(cudaMemset(h->d_xcounter, 0, sizeof(unsigned)));
  CK(cudaMalloc(&h->d_xerr, sizeof(int)));
  CK(cudaMemset(h->d_xerr, 0, sizeof(int)));
  h->xd.rank = rank;
  h->xd.world = world;
  return SB_OK;
}

int sb_xchg_create(sb_handle* h, int rank, int world, void* handle_out) {
  int rc = use_device(h);
  if (rc) return rc;
  if (world < 1 || world > kMaxRanks || rank < 0 || rank >= world)
    return fail(SB_ERR_ARG, "rank %d / world %d outside 0..%d", rank, world, kMaxRanks);
  if (!handle_out) return fail(SB_ERR_ARG, "handle_out is null");
  if ((rc = create_mailbox(h, rank, world))) return rc;
  cudaIpcMemHandle_t hdl;
  CK(cudaIpcGetMemHandle(&hdl, h->xd.local));
  static_assert(sizeof(hdl) == SB_IPC_HANDLE_BYTES, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle_out, &hdl, sizeof(hdl));
  h->xchg_created = true;
  return SB_OK;
}

int sb_xchg_connect(sb_handle* h, const void* handles) {
  int rc = use_device(h);
  if (rc) return rc;
  if (!h->xchg_created) return fail(SB_ERR_STATE, "sb_xchg_create has not been called");
  if (!handles) return fail(SB_ERR_ARG, "handles is null");
  const char* hp = static_cast<const char*>(handles);
  for (int r = 0; r < h->xd.world; ++r) {
    if (r == h->xd.rank) {
      h->xd.peer[r] = h->xd.local;
      continue;
    }
    cudaIpcMemHandle_t hdl;
    memcpy(&hdl, hp + static_cast<size_t>(r) * SB_IPC_HANDLE_BYTES, sizeof(hdl));
    void* p = nullptr;
    cudaError_t e = cudaIpcOpenMemHandle(&p, hdl, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return fail(SB_ERR_CUDA, "cudaIpcOpenMemHandle(rank %d) failed: %s", r, cudaGetErrorString(e));
    }
    h->x_opened[r] = p;
    h->xd.peer[r] = static_cast<unsigned long long*>(p);
  }
  h->xchg_ready = true;
  return SB_OK;
}

int sb_xchg_connect_local(sb_handle** hs, int n) {
  if (!hs || n < 1 || n > kMaxRanks) return fail(SB_ERR_ARG, "need 1..%d handles", kMaxRanks);
  for (int i = 0; i < n; ++i) {
    if (!hs[i]) return fail(SB_ERR_ARG, "handle %d is null", i);
    for (int j = 0; j < i; ++j)
      if (hs[j]->dev.ordinal == hs[i]->dev.ordinal)
        return fail(SB_ERR_ARG, "handles %d and %d share device %d; one handle per device", j, i, hs[i]->dev.ordinal);
  }
  // every handle gets a fresh mailbox on its own device
  for (int i = 0; i < n; ++i) {
    sb_handle* h = hs[i];
    int rc = use_device(h);
    if (rc) return rc;
    CK(cudaStreamSynchronize(h->stream));
    if ((rc = create_mailbox(h, i, n))) return rc;
    h->xchg_created = true;
  }
  // same address space: a peer's mailbox is reachable as soon as peer access is on (no IPC handles)
  for (int i = 0; i < n; ++i) {
    sb_handle* h = hs[i];
    CK(cudaSetDevice(h->dev.ordinal));
    for (int j = 0; j < n; ++j) {
      if (j != i) {
        int can = 0;
        CK(cudaDeviceCanAccessPeer(&can, h->dev.ordinal, hs[j]->dev.ordinal));
        if (!can)
          return fail(SB_ERR_UNSUPPORTED, "device %d cannot map device %d's memory (no NVLink / P2P path)",
                      h->dev.ordinal, hs[j]->dev.ordinal);
        cudaError_t e = cudaDeviceEnablePeerAccess(hs[j]->dev.ordinal, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
        else if (e != cudaSuccess) return fail(SB_ERR_CUDA, "cudaDeviceEnablePeerAccess(%d -> %d): %s", h->dev.ordinal,
                                               hs[j]->dev.ordinal, cudaGetErrorString(e));
      }
      h->xd.peer[j] = hs[j]->xd.local;
    }
    h->xchg_ready = true;
  }
  return SB_OK;
}

int sb_xchg_post(sb_handle* h, const uint64_t* key_dev) {
  int rc = use_device(h);
  if (rc) return rc;
  if (!h->xchg_ready) return fail(SB_ERR_STATE, "sb_xchg_connect has not been called");
  if (!key_dev) return fail(SB_ERR_ARG, "key_dev is null");
  ++h->xseq;
  CK(xchg_post_launch(h->xd, reinterpret_cast<const unsigned long long*>(key_dev), h->xseq, h->stream));
  return SB_OK;
}

int sb_xchg_reduce(sb_handle* h, uint64_t* out_dev, uint64_t* fold_dev) {
  int rc = use_device(h);
  if (rc) return rc;
  if (!h->xchg_ready) return fail(SB_ERR_STATE, "sb_xchg_connect has not been called");
  if (!out_dev) return fail(SB_ERR_ARG, "out_dev is null");
  if (h->xseq == 0) return fail(SB_ERR_STATE, "nothing has been posted yet");
  CK(xchg_reduce_launch(h->xd, h->xseq, reinterpret_cast<unsigned long long*>(out_dev),
                        reinterpret_cast<unsigned long long*>(fold_dev), h->d_xerr, h->stream));
  return SB_OK;
}

int sb_xchg_check(sb_handle* h) {
  int rc = use_device(h);
  if (rc) return rc;
  if (!h->xchg_created) return fail(SB_ERR_STATE, "sb_xchg_create has not been called");
  int err = 0;
  CK(cudaMemcpyAsync(&err, h->d_xerr, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (err) return fail(SB_ERR_CUDA, "peer exchange timed out waiting for a rank's post");
  return SB_OK;
}

// ------------------------------------------------------------------------------------------ search
// Job-indexed opt row (the ABI's encoding) <-> opt by schedule position (position-major populations).
static void opt_to_positions(int J, int pb, const uint8_t* opt, const void* prio, std::vector<uint8_t>* out) {
  out->resize(J);
  for (int i = 0; i < J; ++i) {
    const int j = pb == 1 ? static_cast<const uint8_t*>(prio)[i] : static_cast<const uint16_t*>(prio)[i];
    (*out)[i] = j < J ? opt[j] : 0;
  }
}

static void opt_from_positions(int J, int pb, uint8_t* opt, const void* prio) {
  std::vector<uint8_t> by_pos(opt, opt + J);
  for (int i = 0; i < J; ++i) {
    const int j = pb == 1 ? static_cast<const uint8_t*>(prio)[i] : static_cast<const uint16_t*>(prio)[i];
    if (j < J) opt[j] = by_pos[i];
  }
}

static int search_alloc(SearchState& s, void** p, size_t bytes) {
  if (s.nblocks >= 16) return fail(SB_ERR_NOMEM, "search block table full");
  cudaError_t e = cudaMalloc(p, bytes);
  if (e != cudaSuccess) return fail(SB_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
  s.blocks[s.nblocks++] = *p;
  return SB_OK;
}

// the tables the search's position-major kernel reads: the nominal table, or under the scenario forms the K scenario
// tables (*K = their number)
static const float* search_tables(const sb_handle* h, int* K) {
  const SearchState& s = h->search;
  const bool reduced = (s.p.flags & SB_FLAG_REDUCED) != 0;
  *K = obj_scenario(s.obj.obj) ? h->scen_K : 0;
  if (*K) return reduced ? h->d_scen_min : h->d_scen;
  return reduced ? h->tmin : h->tab;
}

static int search_eval(sb_handle* h, bool cur_rows, long long first, long long count) {
  SearchState& s = h->search;
  if (s.d.pos) {  // position-major rows are only ever scored in place, by their own kernel
    if (!cur_rows) return fail(SB_ERR_STATE, "position-major populations have no proposal rows");
    SearchFuse sf = {};
    sf.cur_mk = s.d.cur_mk;
    const bool reduced = (s.p.flags & SB_FLAG_REDUCED) != 0;
    int K = 0;
    const float* tab = search_tables(h, &K);
    CK(search_pos_launch(h->dev, s.d, tab, s.w, s.due, s.rel, s.pen,
                         (reduced ? 1 : h->S) * kSlots, s.p.flags,
                         s.obj.obj, first, count, true, sf, h->stream, 0, K));
    return SB_OK;
  }
  EvalCall c;
  const uint8_t* ro = (cur_rows ? s.d.cur_o : s.d.prop_o) + first * s.d.stride_o;
  const uint8_t* rp = (cur_rows ? s.d.cur_p : s.d.prop_p) + first * s.d.stride_p;
  int rc = make_call(h, ro, rp, count, s.d.stride_o, s.p.flags, &c);
  if (rc) return rc;
  c.out = (cur_rows ? s.d.cur_mk : s.d.prop_mk) + first;
  c.best_key = s.d.keys;
  c.id_base = static_cast<uint32_t>(s.d.chain_base + static_cast<uint64_t>(first));
  CK(eval_launch(h->dev, c, h->stream, &h->last_path));
  return SB_OK;
}

int sb_search_init(sb_handle* h, const sb_search_params* p, const uint8_t* warm_opt, const void* warm_prio) {
  int rc = use_device(h);
  if (rc) return rc;
  if (h->J == 0) return fail(SB_ERR_STATE, "sb_set_table has not been called");
  if (!p) return fail(SB_ERR_ARG, "params is null");
  if (p->chains < 1 || p->chains > (1ll << 31)) return fail(SB_ERR_ARG, "chains=%lld out of range", (long long)p->chains);
  Objective o;
  if ((rc = check_per_job(h, p->flags, &o))) return rc;
  CK(cudaStreamSynchronize(h->stream));
  SearchState& s = h->search;
  s.ready = false;
  s.p = *p;
  s.obj = o;
  if (s.p.total_rounds < 1) s.p.total_rounds = 1;
  const int J = h->J;
  const int pb = J <= 256 ? 1 : 2;
  SearchDev& d = s.d;
  d.J = J;
  d.pb = pb;
  d.nodes = h->nodes;
  d.chains = p->chains;
  d.chain_base = p->chain_base;
  d.seed = p->seed;
  const int arrays = job_arrays(o.obj, p->flags);
  s.w = job_weights(h, o);
  s.due = job_due(h, o.obj);
  s.rel = job_release(h, p->flags);
  s.pen = job_penalty(h, o.obj);
  d.stride_o = (J + 31) & ~31;  // 32-byte rows: TMA bulk copies for opt, 256-bit streaming loads for prio
  // make stride_p == stride_o * pb so that one element stride describes both (sb_eval contract)
  d.stride_p = d.stride_o * pb;
  const bool reduced = (p->flags & SB_FLAG_REDUCED) != 0;
  if (h->nodes > 1 && !reduced) return fail(SB_ERR_UNSUPPORTED, "multi-node search needs SB_FLAG_REDUCED");
  d.vopt = h->vopt[reduced ? 1 : 0];
  d.nvalid = h->nvalid[reduced ? 1 : 0];
  const size_t P = static_cast<size_t>(d.chains);
  if (s.nblocks > 0 && s.alloc_chains == d.chains && s.alloc_stride_o == d.stride_o && s.alloc_stride_p == d.stride_p) {
    d.cur_o = s.alloc.cur_o; d.cur_p = s.alloc.cur_p; d.prop_o = s.alloc.prop_o; d.prop_p = s.alloc.prop_p;
    d.cur_mk = s.alloc.cur_mk; d.prop_mk = s.alloc.prop_mk; d.keys = s.alloc.keys;
    d.best_o = s.alloc.best_o; d.best_p = s.alloc.best_p;
  } else {
    const SearchDev shape = d;
    const sb_search_params params = s.p;
    free_search(h);
    s.p = params;
    d = shape;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&d.cur_o), P * d.stride_o))) return rc;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&d.cur_p), P * d.stride_p))) return rc;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&d.prop_o), P * d.stride_o))) return rc;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&d.prop_p), P * d.stride_p))) return rc;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&d.cur_mk), P * sizeof(float)))) return rc;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&d.prop_mk), P * sizeof(float)))) return rc;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&d.keys), 2 * sizeof(unsigned long long)))) return rc;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&d.best_o), d.stride_o))) return rc;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&d.best_p), d.stride_p))) return rc;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&s.cand_o), d.stride_o))) return rc;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&s.cand_p), d.stride_p))) return rc;
    if ((rc = search_alloc(s, reinterpret_cast<void**>(&s.tail_counter), sizeof(unsigned)))) return rc;
    s.alloc = d;
    s.alloc_chains = d.chains; s.alloc_stride_o = d.stride_o; s.alloc_stride_p = d.stride_p;
  }
  CK(cudaMemsetAsync(s.tail_counter, 0, sizeof(unsigned), h->stream));
  CK(cudaMemsetAsync(d.keys, 0xff, 2 * sizeof(unsigned long long), h->stream));
  // (the initialisation kernels write whole rows, padding included: no memset of the population)
  // Rows that do not fit in shared memory: keep the population in schedule order and stream both rows.
  const int SGs = (reduced ? 1 : h->S) * kSlots;
  const bool no_fused = (p->flags & HOOK_NO_FUSED) != 0;
  // the scenario forms have no tile kernel: their population is always position-major (check_per_job has held their
  // tables to the position-major kernel's shared memory), or unfused under HOOK_NO_FUSED
  const bool scen = obj_scenario(o.obj);
  const int mode = scen ? 0 : search_round_mode(h->dev, J, SGs, h->nodes, arrays);
  const size_t pos_smem = scen ? scenario_smem(J, SGs, h->scen_K, h->nodes, p->flags, o.obj)
                               : search_pos_smem(J, SGs, h->nodes, 16, arrays);
  d.pos = (!no_fused && mode != 2 && pos_smem <= h->dev.smem_optin) ? 1 : 0;
  if (d.pos) CK(search_init_population_pos(d, h->stream));
  else CK(search_init_population(d, h->stream));
  s.ready = true;
  std::vector<uint8_t> by_pos;
  if (warm_opt && warm_prio) {
    if (d.pos) {
      opt_to_positions(J, pb, warm_opt, warm_prio, &by_pos);
      warm_opt = by_pos.data();
    }
    CK(cudaMemsetAsync(s.cand_o, 0, d.stride_o, h->stream));
    CK(cudaMemsetAsync(s.cand_p, 0, d.stride_p, h->stream));
    CK(cudaMemcpyAsync(s.cand_o, warm_opt, J, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(s.cand_p, warm_prio, static_cast<size_t>(J) * pb, cudaMemcpyHostToDevice, h->stream));
    CK(search_inject(d, s.cand_o, s.cand_p, 0, 1, h->stream));
  }
  if ((rc = search_eval(h, true, 0, d.chains))) return rc;
  CK(search_keep_best(d, true, h->stream));
  unsigned long long key = 0;
  CK(cudaMemcpyAsync(&key, d.keys, sizeof(key), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  uint32_t bits = static_cast<uint32_t>(key >> 32);
  float mk;
  memcpy(&mk, &bits, 4);
  // the temperature unit: the incumbent's makespan, or its mean completion time (the sum / J; weighted: the weighted
  // sum / the sum of the weights, the same fp32 value for unit weights), so that t_start / t_end mean the same
  // fraction of a typical score difference under every objective
  const bool weighted = o.weighted;
  const float per = weighted ? static_cast<float>(h->w_sum) : static_cast<float>(J);
  // The completion penalty keeps this completion unit, with no sum of penalties added: in a front the penalties are
  // a barrier that the warm-started incumbent already clears, and must not heat the search past it.  With every p = 0
  // it is the completion unit bit for bit (a starting point, not a measured choice, DESIGN §3)
  // The tardiness scenario forms take the tardiness unit: the incumbent's score per unit weight (the worst or the sum
  // over K scenarios of a total, so per job as the sum forms), floored below (a starting point, not a measured choice,
  // DESIGN §3)
  const bool scen_t = o.obj == Obj::WorstTardiness || o.obj == Obj::MeanTardiness;
  s.scale = isfinite(mk) ? ((obj_sum(o.obj) || scen_t) ? mk / per : mk) : 1.0f;
  if (tardiness_form(o.obj) && isfinite(mk)) {
    // tardiness can be 0 or tiny at the incumbent: the unit is at least the weighted mean of each job's smallest
    // proposable runtime, the size of the score change one move makes
    const float* tmin = h->h_tmin.data();
    double move = 0.0, move_max = 0.0, move_sq = 0.0;
    for (int j = 0; j < J; ++j) {
      double lo = HUGE_VAL, lo_any = HUGE_VAL;
      for (int k = 0; k < kSlots; ++k) {
        const float v = tmin[j * kSlots + k];
        if (v < h->sentinel) lo = std::min(lo, static_cast<double>(v));
        if (isfinite(v)) lo_any = std::min(lo_any, static_cast<double>(v));
      }
      if (!isfinite(lo)) lo = lo_any;
      if (isfinite(lo)) {
        const double x = (weighted ? static_cast<double>(h->h_w[j]) : 1.0) * lo;
        move += x;
        move_max = std::max(move_max, x);
        move_sq += x * lo;
      }
    }
    // the maximum tardiness is a max, not a sum: its unit is the incumbent itself (the mean-completion division of
    // SB_FLAG_SUM_COMPLETION does not apply), and at least the largest weighted smallest runtime, the same floor taken
    // as a max.  A starting point, not a measured choice (DESIGN §3)
    if (o.obj == Obj::MaxTardiness) s.scale = std::max(mk, static_cast<float>(move_max));
    // the squared tardiness: the same mean-per-weight unit, with the floor's runtimes squared, sum_j w_j lo_j^2 /
    // sum_j w_j (a starting point, not a measured choice, DESIGN §3)
    else if (o.obj == Obj::SquaredTardiness)
      s.scale = std::max(s.scale, static_cast<float>(move_sq / (weighted ? h->w_sum : static_cast<double>(J))));
    // the late penalty: the tardiness floor with every penalty added, (sum_j w_j lo_j + sum_j p_j) / sum_j w_j,
    // which is the tardiness unit bit for bit when every p = 0 (a starting point, not a measured choice, DESIGN §3)
    else if (o.obj == Obj::LatePenalty)
      s.scale = std::max(s.scale, static_cast<float>((move + h->p_sum) / (weighted ? h->w_sum : static_cast<double>(J))));
    // the mean tardiness scores the sum of K totals: K times the floor of one
    else if (o.obj == Obj::MeanTardiness)
      s.scale = std::max(s.scale, static_cast<float>(h->scen_K * move / (weighted ? h->w_sum : static_cast<double>(J))));
    else s.scale = std::max(s.scale, static_cast<float>(move / (weighted ? h->w_sum : static_cast<double>(J))));
  }
  // the late count moves in steps of one job's weight and is 0 at many incumbents: its unit is the count of every job,
  // sum_j w_j (J with unit weights), so that an uphill move of one mean weight is accepted with e^(-1 / (J t))
  if (o.obj == Obj::LateCount) s.scale = static_cast<float>(weighted ? h->w_sum : static_cast<double>(J));
  s.evaluated = d.chains;
  s.rounds_done = 0;
  s.launches = 0;
  s.fused_ok = d.pos || (!no_fused && mode != 0);
  // incremental rounds: fused kernels, one node, at least two windows (tile kernel: windows of kSnapPos
  // positions; position-major kernel: windows of whole 32-position blocks, at most 32 windows)
  int nwin = (J + kSnapPos - 1) / kSnapPos;
  if (d.pos) {
    const int nout = (J + 31) / 32, wblk = (nout + 31) / 32;
    nwin = (nout + wblk - 1) / wblk;
  }
  s.win = s.fused_ok && h->nodes == 1 && nwin >= 2 && nwin <= 32 && !(p->flags & HOOK_ROUND1_MOVES);
  // the scenario forms score every proposal from position 0, as HOOK_NO_INCREMENTAL does (K snapshot sets per window
  // boundary are not kept)
  s.inc = s.win && !(p->flags & HOOK_NO_INCREMENTAL) && !scen;
  s.verify = s.inc && (p->flags & HOOK_VERIFY_INCREMENTAL);
  // automatic cadence: resampling is nearly free inside the tile kernel; elsewhere it is a full copy of the
  // population and ends a launch (an incremental launch starts with one unmodified pass, so longer is better)
  if (s.p.resample_every < 0) s.p.resample_every = (s.fused_ok && !d.pos) ? 2 : (s.inc ? 8 : 4);
  if (s.inc) {
    const size_t need = static_cast<size_t>((d.chains + 31) / 32) * (nwin - 1) * 2 * 9 * 32 * sizeof(float);
    if (s.snap_bytes < need) {
      if (s.snap) {  // grow: drop the old block from the table
        for (int i = 0; i < s.nblocks; ++i)
          if (s.blocks[i] == s.snap) { cudaFree(s.snap); s.blocks[i] = s.blocks[--s.nblocks]; break; }
        s.snap = nullptr;
        s.snap_bytes = 0;
      }
      if ((rc = search_alloc(s, reinterpret_cast<void**>(&s.snap), need))) { s.ready = false; return rc; }
      s.snap_bytes = need;
    }
    if (!s.verify_bad && (rc = search_alloc(s, reinterpret_cast<void**>(&s.verify_bad), sizeof(unsigned long long)))) {
      s.ready = false;
      return rc;
    }
    CK(cudaMemsetAsync(s.verify_bad, 0, sizeof(unsigned long long), h->stream));
  }
  return SB_OK;
}

static float round_temperature(const SearchState& s, int round) {
  float frac = static_cast<float>(round - 1) / static_cast<float>(s.p.total_rounds > 1 ? s.p.total_rounds - 1 : 1);
  if (frac > 1.f) frac = 1.f;
  float tf;
  if (s.p.t_start <= 0.f) tf = 0.f;
  else if (s.p.t_end <= 0.f) tf = s.p.t_start * (1.f - frac);
  else tf = s.p.t_start * powf(s.p.t_end / s.p.t_start, frac);
  return tf * s.scale;
}

// rounds [round, round + n) in one launch
static SearchFuse make_fuse(const SearchState& s, int round, int n) {
  SearchFuse sf;
  sf.cur_mk = s.d.cur_mk; sf.cur_o = s.d.cur_o; sf.cur_p = s.d.cur_p;
  sf.vopt = s.d.vopt; sf.nvalid = s.d.nvalid;
  sf.seed = s.d.seed; sf.chain_base = s.d.chain_base; sf.round = round; sf.nodes = s.d.nodes;
  sf.nrounds = n;
  for (int r = 0; r < n; ++r) sf.temperature[r] = round_temperature(s, round + r);
  sf.resample_every = s.p.resample_every > 0 ? s.p.resample_every : 0;
  sf.deal = static_cast<int>(s.launches & 1);
  sf.win = s.win ? 1 : 0;
  sf.win_bias = (s.p.flags & HOOK_WINDOW_BIAS) ? 1 : 0;
  sf.snap = s.inc ? s.snap : nullptr;
  sf.verify_bad = s.verify ? s.verify_bad : nullptr;
  sf.keep.counter = s.tail_counter;
  sf.keep.keys = s.d.keys;
  sf.keep.best_o = s.d.best_o; sf.keep.best_p = s.d.best_p;
  sf.keep.chains = s.d.chains; sf.keep.stride_o = s.d.stride_o; sf.keep.stride_p = s.d.stride_p;
  return sf;
}

// tournament resampling of the whole population: the kernel writes the result to the proposal buffers, which then
// become the current ones
static int resample_population(sb_handle* h) {
  SearchDev& d = h->search.d;
  CK(search_resample(d, h->search.rounds_done, h->stream));
  std::swap(d.cur_o, d.prop_o);
  std::swap(d.cur_p, d.prop_p);
  std::swap(d.cur_mk, d.prop_mk);
  return SB_OK;
}

int sb_search_round(sb_handle* h, int rounds) {
  int rc = use_device(h);
  if (rc) return rc;
  SearchState& s = h->search;
  if (!s.ready) return fail(SB_ERR_STATE, "sb_search_init has not been called");
  const int re = s.p.resample_every > 0 ? s.p.resample_every : 0;
  int left = rounds;
  while (left > 0) {
    const int round = s.rounds_done + 1;
    int n = 1;  // rounds covered by this iteration
    bool fused = false;
    const bool due = re > 0 && round > 1 && (round - 1) % re == 0;  // the population is resampled before this round
    if (s.d.pos) {
      if (due) {
        if ((rc = resample_population(h))) return rc;
      }
      n = std::min(left, kMaxFusedRounds);
      if (re > 0) n = std::min(n, re - (round - 1) % re);  // up to the next resampling point
      SearchFuse sf = make_fuse(s, round, n);
      sf.resample_every = 0;
      const bool reduced = (s.p.flags & SB_FLAG_REDUCED) != 0;
      int K = 0;
      const float* tab = search_tables(h, &K);
      CK(search_pos_launch(h->dev, s.d, tab, s.w, s.due, s.rel, s.pen,
                         (reduced ? 1 : h->S) * kSlots, s.p.flags,
                           s.obj.obj, 0, s.d.chains, false, sf, h->stream, 0, K));  // keeps the incumbent in its tail
      fused = true;
    } else if (s.fused_ok) {
      EvalCall c;
      if ((rc = make_call(h, s.d.cur_o, s.d.cur_p, s.d.chains, s.d.stride_o, s.p.flags, &c))) return rc;
      c.best_key = s.d.keys;
      c.id_base = static_cast<uint32_t>(s.d.chain_base);
      n = std::min(left, kMaxFusedRounds);
      const SearchFuse sf = make_fuse(s, round, n);  // resamples inside the kernel
      cudaError_t e = search_round_launch(h->dev, c, sf, h->stream);
      if (e == cudaSuccess) {
        fused = true;  // an improving proposal is always accepted, so it is in cur: the kernel's tail saves it
        ++s.launches;
      } else if (e != cudaErrorNotSupported) {
        return fail(SB_ERR_CUDA, "fused search round failed: %s", cudaGetErrorString(e));
      } else {
        cudaGetLastError();
        s.fused_ok = false;
        n = 1;
      }
    }
    if (!fused) {
      if (due) {
        if ((rc = resample_population(h))) return rc;
      }
      CK(search_propose(s.d, round, h->stream));
      if ((rc = search_eval(h, false, 0, s.d.chains))) return rc;
      CK(search_keep_best(s.d, false, h->stream));
      CK(search_accept(s.d, round, round_temperature(s, round), h->stream));
    }
    s.rounds_done = round + n - 1;
    s.evaluated += s.d.chains * n;
    left -= n;
  }
  return SB_OK;
}

int sb_search_best_key_ptr(sb_handle* h, uint64_t** key_dev) {
  if (!h || !key_dev) return fail(SB_ERR_ARG, "null argument");
  if (!h->search.ready) return fail(SB_ERR_STATE, "sb_search_init has not been called");
  *key_dev = reinterpret_cast<uint64_t*>(h->search.d.keys);
  return SB_OK;
}

int sb_search_best(sb_handle* h, uint8_t* opt, void* prio, float* makespan, uint64_t* key_out) {
  int rc = use_device(h);
  if (rc) return rc;
  SearchState& s = h->search;
  if (!s.ready) return fail(SB_ERR_STATE, "sb_search_init has not been called");
  unsigned long long keys[2];
  CK(cudaMemcpyAsync(keys, s.d.keys, sizeof(keys), cudaMemcpyDeviceToHost, h->stream));
  if (opt) CK(cudaMemcpyAsync(opt, s.d.best_o, s.d.J, cudaMemcpyDeviceToHost, h->stream));
  if (prio) CK(cudaMemcpyAsync(prio, s.d.best_p, static_cast<size_t>(s.d.J) * s.d.pb, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  if (s.d.pos && opt) {
    std::vector<uint8_t> pr(static_cast<size_t>(s.d.J) * s.d.pb);
    if (prio) {
      memcpy(pr.data(), prio, pr.size());
    } else {
      CK(cudaMemcpyAsync(pr.data(), s.d.best_p, pr.size(), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
    }
    opt_from_positions(s.d.J, s.d.pb, opt, pr.data());
  }
  if (makespan) {
    uint32_t bits = static_cast<uint32_t>(keys[1] >> 32);
    memcpy(makespan, &bits, 4);
  }
  if (key_out) *key_out = keys[1];
  return SB_OK;
}

int sb_search_resample(sb_handle* h) {
  int rc = use_device(h);
  if (rc) return rc;
  SearchState& s = h->search;
  if (!s.ready) return fail(SB_ERR_STATE, "sb_search_init has not been called");
  return resample_population(h);
}

int sb_search_inject(sb_handle* h, const uint8_t* opt, const void* prio, int64_t first_chain, int copies) {
  int rc = use_device(h);
  if (rc) return rc;
  SearchState& s = h->search;
  if (!s.ready) return fail(SB_ERR_STATE, "sb_search_init has not been called");
  if (!opt || !prio) return fail(SB_ERR_ARG, "opt / prio is null");
  if (copies < 1) return SB_OK;
  if (copies > s.d.chains) copies = static_cast<int>(s.d.chains);
  long long first = first_chain < 0 ? s.d.chains - copies : first_chain;
  if (first + copies > s.d.chains) first = s.d.chains - copies;
  std::vector<uint8_t> by_pos;
  if (s.d.pos) {
    opt_to_positions(s.d.J, s.d.pb, opt, prio, &by_pos);
    opt = by_pos.data();
  }
  CK(cudaMemsetAsync(s.cand_o, 0, s.d.stride_o, h->stream));
  CK(cudaMemsetAsync(s.cand_p, 0, s.d.stride_p, h->stream));
  CK(cudaMemcpyAsync(s.cand_o, opt, s.d.J, cudaMemcpyHostToDevice, h->stream));
  CK(cudaMemcpyAsync(s.cand_p, prio, static_cast<size_t>(s.d.J) * s.d.pb, cudaMemcpyHostToDevice, h->stream));
  CK(search_inject(s.d, s.cand_o, s.cand_p, first, copies, h->stream));
  if ((rc = search_eval(h, true, first, copies))) return rc;
  CK(search_keep_best(s.d, true, h->stream));
  CK(cudaStreamSynchronize(h->stream));  // opt / prio are caller memory: do not return with copies in flight
  s.evaluated += copies;
  return SB_OK;
}

// Moore-Hodgson's repair of a seed order for the late count.  The on-time sequence (at first `order`) is list-scheduled
// on the host in float64 by the device's rule: job j takes the k = col[j] + 1 slots of node[j] that are free first,
// starts when the k-th is free (and not before its release r[j]), holds them for rt[j] (ceil(rt[j]) with integer
// starts) and completes at start + rt[j].  At the first job that completes after its due date d[j], the job with the
// largest k * rt / w among it and the jobs before it (the later one on ties) leaves the sequence for a late list, and
// the schedule is resumed from that job's position; until no job of the sequence is late.  The order becomes the
// on-time sequence followed by the late list in `order`'s order.  One gang size, one node and unit weights make it
// Moore-Hodgson's algorithm, which minimises the number of late jobs; otherwise it is a heuristic.  An order without a
// late job is unchanged.  search.lpt_seeds restates it.
static void moore_hodgson(std::vector<int>& order, const std::vector<int>& col, const std::vector<double>& rt,
                          const std::vector<int>& node, int nodes, const std::vector<float>* w,
                          const std::vector<float>& d, const std::vector<float>* r, bool integer_starts) {
  const int J = static_cast<int>(order.size());
  const size_t state = static_cast<size_t>(nodes) * kSlots;  // the slots' free times, ascending per node
  std::vector<double> snap((static_cast<size_t>(J) + 1) * state, 0.0);  // snap[q]: before sequence position q
  std::vector<int> seq(order), late_list;
  std::vector<int> pos(J);
  for (int q = 0; q < J; ++q) pos[order[q]] = q;
  auto ratio = [&](int j) { return (col[j] + 1) * rt[j] / (w ? static_cast<double>((*w)[j]) : 1.0); };
  size_t q = 0;
  while (q < seq.size()) {
    const int j = seq[q];
    double* cur = snap.data() + (q + 1) * state;
    std::copy(snap.data() + q * state, snap.data() + (q + 1) * state, cur);
    double* f = cur + static_cast<size_t>(node[j]) * kSlots;
    const int k = col[j] + 1;
    double st = f[k - 1];
    if (r) st = std::max(st, static_cast<double>((*r)[j]));
    const double v = st + (integer_starts ? ceil(rt[j]) : rt[j]);
    for (int g = 0; g < k; ++g) f[g] = v;
    std::sort(f, f + kSlots);
    if (st + rt[j] > static_cast<double>(d[j])) {
      size_t out = 0;
      double best = -HUGE_VAL;
      for (size_t p = 0; p <= q; ++p)
        if (ratio(seq[p]) >= best) { best = ratio(seq[p]); out = p; }
      late_list.push_back(seq[out]);
      seq.erase(seq.begin() + static_cast<long>(out));
      q = out;
      continue;
    }
    ++q;
  }
  if (late_list.empty()) return;
  std::sort(late_list.begin(), late_list.end(), [&](int a, int b) { return pos[a] < pos[b]; });
  seq.insert(seq.end(), late_list.begin(), late_list.end());
  order = seq;
}

int sb_search_seed_lpt(sb_handle* h) {
  int rc = use_device(h);
  if (rc) return rc;
  SearchState& s = h->search;
  if (!s.ready) return fail(SB_ERR_STATE, "sb_search_init has not been called");
  const int J = h->J, nodes = h->nodes;
  const bool reduced = (s.p.flags & SB_FLAG_REDUCED) != 0;
  const float* tmin = h->h_tmin.data();
  const Obj obj = s.obj.obj;
  // shortest first: the order that favours the sum (and, below, the tie-break of the due-date orders)
  // the scenario forms seed as their step's form does, on the nominal table: the makespan's orders, or the tardiness
  // form's EDD orders (which with every due date +0 are the SPT / WSPT orders of the completion forms)
  const bool spt = step_obj(obj) != Obj::Makespan && obj != Obj::TailMakespan;
  // weighted sum: Smith's rule (WSPT), ascending rt / w; with unit weights exactly the SPT order
  const bool wspt = spt && s.obj.weighted;
  // the due-date objectives: earliest due date first (EDD), ties by rt / w (rt with unit weights), then by job index;
  // the maximum lateness the same unit-weight EDD orders (Jackson's rule, optimal for L_max on one machine).  The
  // completion penalty keeps the completion orders: its due dates are a barrier on the completion time (one cap for
  // every job in a front), and WSPT is what lowers the sum below it
  const bool edd = obj_due(obj) && obj != Obj::CompletionPenalty;
  const bool rel = (s.p.flags & SB_FLAG_RELEASE) != 0;
  // the late count: each EDD order repaired by Moore-Hodgson's rule (see moore_hodgson)
  const bool late = obj == Obj::LateCount;
  const double INF = HUGE_VAL;
  // usable cells: the ones the search proposes (k_build_valid), per job: those below the sentinel threshold, and for
  // a job with none only its cheapest finite cell (the first minimum; column 0 if it has no finite cell)
  std::vector<double> usable(static_cast<size_t>(J) * kSlots);
  for (int j = 0; j < J; ++j) {
    bool any = false;
    float best = INFINITY;
    int best_c = 0;
    for (int c = 0; c < kSlots; ++c) {
      const float v = tmin[j * kSlots + c];
      usable[j * kSlots + c] = (v < h->sentinel) ? v : INF;
      any = any || (v < h->sentinel);
      if (v < best) { best = v; best_c = c; }
    }
    if (!any) usable[j * kSlots + best_c] = best;
  }
  const long long chains = s.d.chains;
  const long long per = std::max<long long>(1, chains / 8);
  std::vector<int> col(J), order(J);
  std::vector<double> rt(J), weight(J);
  std::vector<uint8_t> opt(J);
  std::vector<uint16_t> prio16(J);
  std::vector<uint8_t> prio8(J);
  const double area_weights[3] = {0.0, 1.0, 0.5};
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < J; ++j) {
      int best = 0;
      double bc = usable[j * kSlots] * pow(1.0, area_weights[i]);
      for (int c = 1; c < kSlots; ++c) {
        const double cost = usable[j * kSlots + c] * pow(c + 1.0, area_weights[i]);
        if (cost < bc) { bc = cost; best = c; }
      }
      col[j] = best;
      rt[j] = usable[j * kSlots + best];
      weight[j] = rt[j] * sqrt(best + 1.0);
      order[j] = j;
    }
    if (edd) {
      for (int j = 0; j < J; ++j) weight[j] = wspt ? rt[j] / static_cast<double>(h->h_w[j]) : rt[j];
      std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
        if (h->h_d[a] != h->h_d[b]) return h->h_d[a] < h->h_d[b];
        return weight[a] < weight[b];
      });
    } else if (wspt) {
      for (int j = 0; j < J; ++j) weight[j] = rt[j] / static_cast<double>(h->h_w[j]);
      std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return weight[a] < weight[b]; });
    } else if (spt) std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return rt[a] < rt[b]; });
    else std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return weight[a] > weight[b]; });
    if (rel) {  // release dates: ascending release first, the objective's order among jobs released together
      const std::vector<float>& r = (s.p.flags & SB_FLAG_INTEGER_STARTS) ? h->h_rc : h->h_r;
      std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return r[a] < r[b]; });
    }
    std::vector<double> load(nodes, 0.0);
    for (int j = 0; j < J; ++j) opt[j] = static_cast<uint8_t>(col[j]);
    if (nodes > 1) {
      for (int q = 0; q < J; ++q) {
        const int j = order[q];
        int n = 0;
        for (int m = 1; m < nodes; ++m)
          if (load[m] < load[n]) n = m;
        load[n] += rt[j] * (col[j] + 1);
        opt[j] = static_cast<uint8_t>(col[j] | (n << 3));
      }
    } else if (!reduced) {
      for (int j = 0; j < J; ++j) opt[j] = static_cast<uint8_t>((h->h_args[j * kSlots + col[j]] << 3) | col[j]);
    }
    if (late) {
      std::vector<int> node(J, 0);
      if (nodes > 1)
        for (int j = 0; j < J; ++j) node[j] = opt[j] >> 3;
      const std::vector<float>* r = rel ? ((s.p.flags & SB_FLAG_INTEGER_STARTS) ? &h->h_rc : &h->h_r) : nullptr;
      moore_hodgson(order, col, rt, node, nodes, s.obj.weighted ? &h->h_w : nullptr, h->h_d, r,
                    (s.p.flags & SB_FLAG_INTEGER_STARTS) != 0);
    }
    for (int q = 0; q < J; ++q) { prio8[q] = static_cast<uint8_t>(order[q]); prio16[q] = static_cast<uint16_t>(order[q]); }
    const long long first = std::min<long long>(i * per, std::max<long long>(0, chains - per));
    const int copies = static_cast<int>(std::min<long long>(per, chains));
    const void* pr = s.d.pb == 1 ? static_cast<const void*>(prio8.data()) : static_cast<const void*>(prio16.data());
    if ((rc = sb_search_inject(h, opt.data(), pr, first, copies))) return rc;
  }
  return SB_OK;
}

// The search loop shared by sb_search_run (n = 1) and sb_search_run_multi (one handle per device of this
// process): every device runs its own population; after each group of rounds the devices exchange ONE uint64
// over NVLink peer memory (publish in the own mailbox, fold of all mailboxes by a one-warp kernel), the host
// reads the folded key of every device with one copy each and applies the stopping rules.
static int search_run_impl(sb_handle** hs, int n, const sb_search_params* p, const sb_search_control* c,
                           const uint8_t* warm_opt, const void* warm_prio, uint8_t* opt_out, void* prio_out,
                           sb_search_result* result) {
  if (!hs || !p || !c) return fail(SB_ERR_ARG, "null argument");
  if (n < 1 || n > kMaxRanks) return fail(SB_ERR_ARG, "need 1..%d handles", kMaxRanks);
  if (c->rounds < 1 || c->sync_every < 1 || c->resample_every < -1 || c->patience < 0)
    return fail(SB_ERR_ARG, "rounds / sync_every must be >= 1, resample_every >= -1, patience >= 0");
  for (int i = 0; i < n; ++i)
    if (!hs[i]) return fail(SB_ERR_ARG, "handle %d is null", i);
  const auto t0 = std::chrono::steady_clock::now();
  auto elapsed = [&]() { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); };
  int rc;
  if (n > 1) {
    bool wired = true;
    for (int i = 0; i < n; ++i) wired = wired && hs[i]->xchg_ready && hs[i]->xd.world == n && hs[i]->xd.rank == i;
    if (!wired && (rc = sb_xchg_connect_local(hs, n))) return rc;
  }
  // population set-up (allocation on first use, initialisation, first scoring, LPT seeds: several host
  // synchronisations per device) runs on one host thread per device — done one device after the other it
  // dominates a short multi-device search
  auto setup = [&](int i) -> int {
    sb_search_params pp = *p;
    pp.total_rounds = c->rounds;
    pp.resample_every = c->resample_every;
    pp.chain_base = p->chain_base + static_cast<uint64_t>(i) * static_cast<uint64_t>(p->chains);
    // the warm start goes to device 0 only: one copy of the previous plan is enough, the rest stays diverse
    int r = sb_search_init(hs[i], &pp, i == 0 ? warm_opt : nullptr, i == 0 ? warm_prio : nullptr);
    if (r == SB_OK && c->heuristic_seeds) r = sb_search_seed_lpt(hs[i]);
    return r;
  };
  if (n == 1) {
    if ((rc = setup(0))) return rc;
  } else {
    std::vector<int> rcs(n, SB_OK);
    std::vector<std::string> msgs(n);
    std::vector<std::thread> workers;
    for (int i = 0; i < n; ++i)
      workers.emplace_back([&, i]() {
        rcs[i] = setup(i);
        if (rcs[i] != SB_OK) msgs[i] = g_err;  // the message lives in the worker's thread-local buffer
      });
    for (auto& w : workers) w.join();
    for (int i = 0; i < n; ++i)
      if (rcs[i] != SB_OK) return fail(rcs[i], "device %d: %s", hs[i]->dev.ordinal, msgs[i].c_str());
  }
  std::vector<unsigned long long> hk(n, ~0ull), hres(2 * static_cast<size_t>(n), 0ull);
  std::vector<int> herr(n, 0);
  // one exchange + host read: returns the best key over all devices
  auto exchange = [&](unsigned long long* best) -> int {
    if (n == 1) {
      sb_handle* h = hs[0];
      CK(cudaSetDevice(h->dev.ordinal));
      CK(cudaMemcpyAsync(&hk[0], h->search.d.keys + 1, sizeof(hk[0]), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      *best = hk[0];
      return SB_OK;
    }
    // per device: ONE kernel (publish the key of the saved incumbent, then fold every device's mailbox) and one
    // 16-byte read-back of {folded key, error flag}
    // Every device's kernel must be QUEUED before the host waits on any of them: a kernel spins until all
    // devices have published, and a device-to-host copy into pageable memory blocks the host until the stream
    // has drained (copy right behind the launch = device 0 waits for a kernel that was never launched:
    // the first version of this loop timed out exactly so).
    for (int i = 0; i < n; ++i) {
      sb_handle* h = hs[i];
      CK(cudaSetDevice(h->dev.ordinal));
      ++h->xseq;
      CK(xchg_post_reduce_launch(h->xd, h->search.d.keys + 1, h->xseq, h->d_scratch + 2, h->stream));
    }
    for (int i = 0; i < n; ++i) {
      sb_handle* h = hs[i];
      CK(cudaSetDevice(h->dev.ordinal));
      CK(cudaMemcpyAsync(&hres[2 * i], h->d_scratch + 2, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
      CK(cudaStreamSynchronize(h->stream));
      hk[i] = hres[2 * i];
      herr[i] = hres[2 * i + 1] != 0;
    }
    for (int i = 0; i < n; ++i) {
      if (herr[i]) return fail(SB_ERR_CUDA, "peer exchange timed out on device %d waiting for a device's key", hs[i]->dev.ordinal);
      if (hk[i] != hk[0]) return fail(SB_ERR_CUDA, "devices disagree on the folded key (%llx on %d, %llx on %d)", hk[0],
                                      hs[0]->dev.ordinal, hk[i], hs[i]->dev.ordinal);
    }
    *best = hk[0];
    return SB_OK;
  };
  auto evaluated = [&]() {
    long long e = 0;
    for (int i = 0; i < n; ++i) e += hs[i]->search.evaluated;
    return e;
  };
  int hist = 0;
  auto record = [&](unsigned long long key) {
    if (c->history_cap > 0 && hist < c->history_cap) {
      uint32_t bits = static_cast<uint32_t>(key >> 32);
      float mk;
      memcpy(&mk, &bits, 4);
      if (c->history_wall_s) c->history_wall_s[hist] = elapsed();
      if (c->history_evaluated) c->history_evaluated[hist] = evaluated();
      if (c->history_makespan) c->history_makespan[hist] = mk;
      ++hist;
    }
  };
  if (n > 1) {
    // every device has finished its initialisation (first launches load their kernels) before the first
    // bounded wait on a peer's mailbox
    for (int i = 0; i < n; ++i) {
      CK(cudaSetDevice(hs[i]->dev.ordinal));
      CK(cudaStreamSynchronize(hs[i]->stream));
    }
  }
  unsigned long long best = 0, key = 0;
  if ((rc = exchange(&best))) return rc;
  record(best);
  // a score of +0 (key bits 0) cannot be beaten
  const bool stop_at_zero = tardiness_form(hs[0]->search.obj.obj);
  int done = 0, stale = 0, reason = (stop_at_zero && (best >> 32) == 0) ? 3 : 0;
  bool first_group = true;
  while (reason == 0 && done < c->rounds) {
    const int step = std::min(c->sync_every, c->rounds - done);
    for (int i = 0; i < n; ++i)
      if ((rc = sb_search_round(hs[i], step))) return rc;  // asynchronous; resamples on its own cadence
    if (n > 1 && first_group) {
      for (int i = 0; i < n; ++i) {
        CK(cudaSetDevice(hs[i]->dev.ordinal));
        CK(cudaStreamSynchronize(hs[i]->stream));
      }
      first_group = false;
    }
    done += step;
    if ((rc = exchange(&key))) return rc;
    if (key < best) { best = key; stale = 0; } else { stale += step; }
    record(best);
    uint32_t bits = static_cast<uint32_t>(best >> 32);
    float mk;
    memcpy(&mk, &bits, 4);
    if (c->time_budget_s > 0 && elapsed() > c->time_budget_s) { reason = 1; break; }
    if (c->patience > 0 && stale >= c->patience) { reason = 2; break; }
    if (c->target_makespan > 0 && mk <= c->target_makespan) { reason = 3; break; }
    if (stop_at_zero && (best >> 32) == 0) { reason = 3; break; }
  }
  // the incumbent lives on the device that owns the chain id in the key
  int owner = 0;
  if (n > 1) {
    const uint64_t id = best & 0xffffffffull;
    const uint64_t rel = (id - (p->chain_base & 0xffffffffull)) & 0xffffffffull;
    owner = static_cast<int>(rel / static_cast<uint64_t>(p->chains));
    if (owner >= n) return fail(SB_ERR_STATE, "best key %llx names chain %llu outside the %d populations", best,
                                static_cast<unsigned long long>(rel), n);
  }
  float mk = 0.f;
  uint64_t k64 = 0;
  if ((rc = sb_search_best(hs[owner], opt_out, prio_out, &mk, &k64))) return rc;
  if (n > 1 && k64 != best)
    return fail(SB_ERR_STATE, "device %d saved key %llx, the exchange says %llx", hs[owner]->dev.ordinal,
                static_cast<unsigned long long>(k64), best);
  if (c->history_len) *c->history_len = hist;
  if (result) {
    result->makespan = mk;
    result->key = k64;
    result->evaluated = evaluated();
    result->rounds = done;
    result->stop_reason = reason;
    result->wall_s = elapsed();
  }
  return SB_OK;
}

int sb_search_run(sb_handle* h, const sb_search_params* p, const sb_search_control* c, const uint8_t* warm_opt,
                  const void* warm_prio, uint8_t* opt_out, void* prio_out, sb_search_result* result) {
  if (!h) return fail(SB_ERR_ARG, "null argument");
  return search_run_impl(&h, 1, p, c, warm_opt, warm_prio, opt_out, prio_out, result);
}

int sb_search_run_multi(sb_handle** handles, int n, const sb_search_params* p, const sb_search_control* c,
                        const uint8_t* warm_opt, const void* warm_prio, uint8_t* opt_out, void* prio_out,
                        sb_search_result* result) {
  return search_run_impl(handles, n, p, c, warm_opt, warm_prio, opt_out, prio_out, result);
}

int sb_search_wave(sb_handle* h, unsigned flags, int64_t* chains) {
  if (!h || !chains) return fail(SB_ERR_ARG, "null argument");
  if (h->J == 0) return fail(SB_ERR_STATE, "sb_set_table has not been called");
  const bool reduced = (flags & SB_FLAG_REDUCED) != 0;
  const int SG = (reduced ? 1 : h->S) * kSlots;
  const int pb = h->J <= 256 ? 1 : 2;
  Objective o;
  if (int rc = decode_objective(flags, &o)) return rc;
  const int arrays = job_arrays(o.obj, flags);
  int warps = 0;
  TilePlan tp;
  if (obj_scenario(o.obj)) {  // the position-major kernel, 16 warps per CTA (sb_search_init)
    warps = 16;
  } else if (search_round_mode(h->dev, h->J, SG, h->nodes, arrays) == 2) {
    plan_tiles(h->dev, h->J, SG, pb, false, h->nodes, &tp, false, arrays);
    warps = tp.warps;
  } else if (search_pos_smem(h->J, SG, h->nodes, 16, arrays) <= h->dev.smem_optin) {
    warps = 16;
  } else {  // unfused rounds: the evaluation kernel's own plan (1 warp stands for the generic kernel's 128-thread CTAs)
    warps = plan_tiles(h->dev, h->J, SG, pb, true, h->nodes, &tp, false, arrays);
    if (warps < 1) warps = 4;
  }
  *chains = static_cast<int64_t>(warps) * 32 * h->dev.sm_count;
  return SB_OK;
}

int sb_search_validate(sb_handle* h, int64_t* bad_rows) {
  int rc = use_device(h);
  if (rc) return rc;
  SearchState& s = h->search;
  if (!s.ready) return fail(SB_ERR_STATE, "sb_search_init has not been called");
  if (!bad_rows) return fail(SB_ERR_ARG, "bad_rows is null");
  EvalCall c;
  if ((rc = make_call(h, s.d.cur_o, s.d.cur_p, s.d.chains, s.d.stride_o, s.p.flags & (SB_FLAG_REDUCED | SB_FLAG_INTEGER_STARTS), &c)))
    return rc;
  CK(cudaMemsetAsync(h->d_scratch, 0, sizeof(unsigned long long), h->stream));
  CK(validate_launch(h->dev, c, h->d_scratch, h->stream, s.d.pos != 0));
  unsigned long long bad = 0;
  CK(cudaMemcpyAsync(&bad, h->d_scratch, sizeof(bad), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  *bad_rows = static_cast<int64_t>(bad);
  return SB_OK;
}

int sb_search_verify_count(sb_handle* h, uint64_t* mismatches) {
  int rc = use_device(h);
  if (rc) return rc;
  if (!mismatches) return fail(SB_ERR_ARG, "mismatches is null");
  SearchState& s = h->search;
  if (!s.ready) return fail(SB_ERR_STATE, "sb_search_init has not been called");
  *mismatches = 0;
  if (!s.verify_bad) return SB_OK;
  unsigned long long v = 0;
  CK(cudaMemcpyAsync(&v, s.verify_bad, sizeof(v), cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  *mismatches = v;
  return SB_OK;
}

int sb_debug_tile_options(sb_handle* h, unsigned options) {
  if (!h) return fail(SB_ERR_ARG, "null handle");
  if (options & ~(TILE_DEBUG_TIMING | TILE_DEBUG_ROW_COPIES | TILE_DEBUG_NO_STAGGER))
    return fail(SB_ERR_ARG, "unknown tile debug option 0x%x", options);
  h->tile_debug = options;
  return SB_OK;
}

int sb_debug_tile_wait(sb_handle* h, uint64_t* out) {
  int rc = use_device(h);
  if (rc) return rc;
  if (!out) return fail(SB_ERR_ARG, "out is null");
  unsigned long long v[2] = {0ull, 0ull};
  if (h->d_tile_wait) {
    CK(cudaMemcpyAsync(v, h->d_tile_wait, sizeof(v), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemsetAsync(h->d_tile_wait, 0, sizeof(v), h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  out[0] = v[0];
  out[1] = v[1];
  return SB_OK;
}

int sb_debug_search_population(sb_handle* h, int64_t first, int64_t count, uint8_t* opt, void* prio, float* score,
                               int* layout) {
  int rc = use_device(h);
  if (rc) return rc;
  SearchState& s = h->search;
  if (!s.ready) return fail(SB_ERR_STATE, "sb_search_init has not been called");
  if (first < 0 || count < 0 || first + count > s.d.chains)
    return fail(SB_ERR_ARG, "chains [%lld, %lld) outside the population of %lld", (long long)first,
                (long long)(first + count), (long long)s.d.chains);
  const size_t J = static_cast<size_t>(s.d.J), pbytes = J * s.d.pb;
  // position-major rows need their priorities to come back job-indexed
  std::vector<uint8_t> pr;
  uint8_t* prio_out = static_cast<uint8_t*>(prio);
  if (s.d.pos && opt && !prio_out) {
    pr.resize(static_cast<size_t>(count) * pbytes);
    prio_out = pr.data();
  }
  if (count > 0) {
    if (opt)
      CK(cudaMemcpy2DAsync(opt, J, s.d.cur_o + first * s.d.stride_o, s.d.stride_o, J, count, cudaMemcpyDeviceToHost,
                           h->stream));
    if (prio_out)
      CK(cudaMemcpy2DAsync(prio_out, pbytes, s.d.cur_p + first * s.d.stride_p, s.d.stride_p, pbytes, count,
                           cudaMemcpyDeviceToHost, h->stream));
    if (score)
      CK(cudaMemcpyAsync(score, s.d.cur_mk + first, static_cast<size_t>(count) * sizeof(float), cudaMemcpyDeviceToHost,
                         h->stream));
  }
  CK(cudaStreamSynchronize(h->stream));
  if (s.d.pos && opt)
    for (int64_t c = 0; c < count; ++c) opt_from_positions(s.d.J, s.d.pb, opt + c * J, prio_out + c * pbytes);
  if (layout) *layout = s.d.pos ? 2 : (s.fused_ok ? 1 : 0);
  return SB_OK;
}

int sb_search_is_fused(sb_handle* h) { return (h && h->search.ready && h->search.fused_ok) ? 1 : 0; }

int sb_search_stats(sb_handle* h, int64_t* evaluated, int64_t* rounds_done) {
  if (!h) return fail(SB_ERR_ARG, "null handle");
  if (evaluated) *evaluated = h->search.evaluated;
  if (rounds_done) *rounds_done = h->search.rounds_done;
  return SB_OK;
}

}  // extern "C"
