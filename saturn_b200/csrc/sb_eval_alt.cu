// sb_eval_alt.cu — the evaluation kernel in the shape BASELINE.json's north_star sketches: the GPU-slot
// earliest-free-times of ONE candidate spread over the lanes of a warp and combined with warp shuffles.
//
// It exists to be measured next to the shipped kernel (one candidate per LANE, sb_eval.cu), not to be used:
// SURVEY.md §7 H2 asked for the alternates behind the same ABI with ncu / the clock deciding, and DESIGN.md
// §5.1 only argued by instruction count.  Selected with SB_FLAG_ALT_WARPSCAN; same inputs, bit-identical
// makespans (tests/test_gpu_parity.py); bench.py reports its rate as configs.C4_alt_shape.
//
// Shape: 8 slots = 8 lanes, so a warp carries 4 candidates (lever (i) of SURVEY H2 — one candidate per
// 32-lane warp would leave 24 lanes idle in every instruction below).  The 8 ready-times of a candidate are
// kept SORTED across its 8 lanes (lane g holds the g-th smallest; which physical GPU that is does not affect
// starts or the makespan, as in the shipped kernel).  A job with k GPUs: s = value of lane k-1 (one shuffle),
// the new sorted state of lane i is max(f_i, min(s + hold, f_{i+k})) with f_{i+k} fetched by ONE
// shuffle-down by the run-time distance k — the dynamic shift that costs the lane-per-candidate kernel a
// 24-select barrel shifter is a single instruction here, but it is a SHFL: the SM executes one warp-wide
// shuffle per clock, and the step also needs its look-ups broadcast by shuffle.
// Look-ups are batched: lane g of a group resolves schedule position i0 + g (job id, opt byte, runtime), then
// the 8 dependent steps read them with shuffles — 8 independent gathers in flight per group.
#include "sb_lane.cuh"

namespace sb {

struct AltArgs {
  const float* tab;
  int J, SG;
  const uint8_t* opt;
  const uint8_t* prio;
  long long B;
  long long stride_o, stride_p;
  float* out;
  unsigned long long* best_key;
  uint32_t id_base;
};

template <int PB, bool INT>
__global__ void __launch_bounds__(512) k_eval_groups(const AltArgs a) {
  extern __shared__ __align__(16) uint8_t smem_alt[];
  float* tab_s = reinterpret_cast<float*>(smem_alt);
  const int n = a.J * a.SG;
  for (int i = threadIdx.x; i < n; i += blockDim.x) tab_s[i] = a.tab[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, g = lane & 7;
  const unsigned gmask = 0xffu << (lane & 24);  // the 8 lanes of this candidate
  const long long ngroups = (a.B + 3) / 4 * 4;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const float INF = inf_f();
  for (long long b4 = warp * 4; b4 < ngroups; b4 += warps * 4) {
    const long long b = b4 + (lane >> 3);
    const bool active = b < a.B;
    const long long br = active ? b : a.B - 1;  // idle groups shadow the last candidate: shuffles stay converged
    const uint8_t* orow = a.opt + br * a.stride_o;
    const uint8_t* prow = a.prio + br * a.stride_p;
    float f = 0.f;   // lane g: the g-th smallest ready time of the candidate
    float mk = 0.f;  // running makespan (identical in the 8 lanes)
    for (int i0 = 0; i0 < a.J; i0 += 8) {
      // lane g resolves position i0 + g
      const int i = i0 + g;
      int o = 0;
      float rt = 0.f;
      if (i < a.J) {
        const int j = PB == 1 ? prow[i] : reinterpret_cast<const uint16_t*>(prow)[i];
        o = orow[j];
        rt = tab_s[j * a.SG + o];
      }
      const int nst = min(8, a.J - i0);
      for (int t = 0; t < nst; ++t) {
        const int ot = __shfl_sync(0xffffffffu, o, (lane & 24) | t);
        const float rtt = __shfl_sync(0xffffffffu, rt, (lane & 24) | t);
        const int k = (ot & 7) + 1;
        const float s = __shfl_sync(0xffffffffu, f, (lane & 24) | (k - 1));  // k-th smallest
        float sh = __shfl_down_sync(0xffffffffu, f, k, 8);                    // f_{g+k}; lanes past the end keep their own
        if (g + k > 7) sh = INF;
        const float v = s + (INT ? ceilf(rtt) : rtt);
        f = fmaxf(f, fminf(v, sh));
        mk = fmaxf(mk, INT ? s + rtt : v);
      }
    }
    (void)gmask;
    if (active && g == 0) a.out[b] = mk;
    if (a.best_key != nullptr) {
      // one representative lane per candidate takes part in the fold
      fold_best(a.best_key, active && g == 0, mk, a.id_base + static_cast<uint32_t>(b), lane);
    }
  }
}

cudaError_t eval_alt_launch(const Device& dev, const EvalCall& c, cudaStream_t st) {
  if (c.B <= 0) return cudaSuccess;
  if (c.nodes > 1) return cudaErrorNotSupported;
  const size_t smem = static_cast<size_t>(c.J) * c.SG * 4;
  if (smem > dev.smem_optin) return cudaErrorNotSupported;
  AltArgs a;
  a.tab = c.tab; a.J = c.J; a.SG = c.SG; a.opt = c.opt; a.prio = c.prio; a.B = c.B;
  a.stride_o = c.stride_o; a.stride_p = c.stride_p; a.out = c.out; a.best_key = c.best_key; a.id_base = c.id_base;
  // resident CTAs per SM are bounded by the table copy each of them holds
  const int threads = 512;
  int per_sm = static_cast<int>(dev.smem_optin / (smem + 1024));
  per_sm = per_sm < 1 ? 1 : (per_sm > 4 ? 4 : per_sm);
  const long long need = (c.B + 4 * (threads / 32) - 1) / (4 * (threads / 32));
  const long long cap = static_cast<long long>(dev.sm_count) * per_sm;
  const int grid = static_cast<int>(need < cap ? need : cap);
  const auto kern = with_pb(c.J <= 256 ? 1 : 2, [&](auto PB) {
    return with_bool(c.flags & SB_FLAG_INTEGER_STARTS, [&](auto INT) { return k_eval_groups<PB, INT>; });
  });
  return launch(kern, grid, threads, smem, st, a);
}

}  // namespace sb
