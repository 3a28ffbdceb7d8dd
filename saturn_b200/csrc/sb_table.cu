// sb_table.cu — ingest of the profiled runtime tensor T[J][S][G].
//
// Reference: the solver's only input is task.strategies, flattened at
// saturn/solver/milp.py:77-81 into (gpu_count, runtime) tuples; the strategy axis has already
// been collapsed by the profiler's min-over-executors (saturn/trial_runner/PerformanceEvaluator.py
// :101-115, strict '<' => the first executor attaining the minimum is kept).  Here the
// un-reduced tensor is accepted, laid out canonically for the evaluator (column = gpu_count-1,
// +inf where no option exists) and the same reduction is produced on the device.
#include "sb_internal.h"

namespace sb {

// one thread per (j, s): scatter the G input columns to their gpu-count column.  Columns with the same GPU count
// keep the first one (in input order) that attains their minimum, with its bits: -0.0 and +0.0 compare equal, so the
// sign of a zero comes from the earlier column, whatever min() does with zeros of both signs.  A negative or NaN
// cell sets *bad: the list-scheduling step needs every hold >= 0 (-0.0 counts as zero; +inf and sentinels are
// legal), and a NaN is no runtime.
__global__ void k_canon_table(const float* __restrict__ T, int J, int S, int G, uint64_t gcount_packed,
                              float* __restrict__ tab, unsigned long long* __restrict__ bad) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= J * S) return;
  float col[kSlots];
#pragma unroll
  for (int c = 0; c < kSlots; ++c) col[c] = inf_f();
  for (int g = 0; g < G; ++g) {
    const int k = static_cast<int>((gcount_packed >> (8 * g)) & 0xff);
    const float v = T[static_cast<size_t>(idx) * G + g];
    if (!(v >= 0.f)) *bad = 1ull;
#pragma unroll
    for (int c = 0; c < kSlots; ++c)
      if (c == k - 1 && v < col[c]) col[c] = v;
  }
#pragma unroll
  for (int c = 0; c < kSlots; ++c) tab[static_cast<size_t>(idx) * kSlots + c] = col[c];
}

// one thread per (j, c): min over strategies, first minimum wins
__global__ void k_reduce_table(const float* __restrict__ tab, int J, int S, float* __restrict__ tmin,
                               uint8_t* __restrict__ args) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= J * kSlots) return;
  const int j = idx / kSlots, c = idx % kSlots;
  float best = inf_f();
  int arg = 0;
  for (int s = 0; s < S; ++s) {
    const float v = tab[(static_cast<size_t>(j) * S + s) * kSlots + c];
    if (v < best) {
      best = v;
      arg = s;
    }
  }
  tmin[idx] = best;
  args[idx] = static_cast<uint8_t>(arg);
}

cudaError_t build_table_launch(const float* T, int J, int S, int G, uint64_t gcount_packed, float* tab, float* tmin,
                               uint8_t* args, unsigned long long* bad, cudaStream_t st) {
  const int n1 = J * S;
  k_canon_table<<<(n1 + 127) / 128, 128, 0, st>>>(T, J, S, G, gcount_packed, tab, bad);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const int n2 = J * kSlots;
  k_reduce_table<<<(n2 + 127) / 128, 128, 0, st>>>(tab, J, S, tmin, args);
  return cudaGetLastError();
}

// one thread per (k, j, c): scenario k's cell, one fp32 product rounded to nearest (f > 0 finite: +inf stays +inf, a
// sentinel scales like any runtime).  One factor per job scales every option of the job alike, so the reduced
// table's arg-min is the same in every scenario and the factor may scale the reduced table directly.
__global__ void k_scale_tables(const float* __restrict__ tab, int J, int SG, const float* __restrict__ f, int K,
                               float* __restrict__ out) {
  const long long n = static_cast<long long>(K) * J * SG;
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const long long cells = static_cast<long long>(J) * SG;
  const int k = static_cast<int>(idx / cells);
  const long long jc = idx % cells;
  const int j = static_cast<int>(jc / SG);
  out[idx] = __fmul_rn(f[static_cast<size_t>(k) * J + j], tab[jc]);
}

cudaError_t scale_tables_launch(const float* tab, int J, int SG, const float* f, int K, float* out, cudaStream_t st) {
  const long long n = static_cast<long long>(K) * J * SG;
  k_scale_tables<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(tab, J, SG, f, K, out);
  return cudaGetLastError();
}

// Valid option list per job for the search's proposals.  Only non-dominated cells are proposed:
// for each gpu count the fastest strategy (a slower strategy with the same footprint can never
// improve the optimum), and only cells below the reference's sentinel runtimes (1e6 "not
// profiled", 1e8 "every executor failed", PerformanceEvaluator.py:99,106 — selecting those would
// hand the executor a Strategy whose executor is None).  A job whose every cell is a sentinel
// keeps its cheapest finite cell so that it can still be scheduled.  One thread per job.
__global__ void k_build_valid(const float* __restrict__ tmin, const uint8_t* __restrict__ args, int J, int reduced,
                              float sentinel, uint8_t* __restrict__ vopt, int* __restrict__ nvalid) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= J) return;
  int n = 0;
  float best = inf_f();
  int best_o = 0;
  for (int c = 0; c < kSlots; ++c) {
    const float v = tmin[j * kSlots + c];
    const int o = reduced ? c : ((static_cast<int>(args[j * kSlots + c]) << 3) | c);
    if (v < best) {
      best = v;
      best_o = o;
    }
    if (v < sentinel) vopt[j * kSlots + n++] = static_cast<uint8_t>(o);
  }
  if (n == 0) vopt[j * kSlots + n++] = static_cast<uint8_t>(best_o);
  nvalid[j] = n;
}

cudaError_t build_valid_launch(const float* tmin, const uint8_t* args, int J, int reduced, float sentinel, uint8_t* vopt,
                               int* nvalid, cudaStream_t st) {
  k_build_valid<<<(J + 127) / 128, 128, 0, st>>>(tmin, args, J, reduced, sentinel, vopt, nvalid);
  return cudaGetLastError();
}

}  // namespace sb
