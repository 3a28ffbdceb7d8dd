// sb_common.cuh — shared device helpers for the SPASE candidate evaluator (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/saturn_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "saturn_b200 kernels target sm_90a (H100) only"
#endif

namespace sb {

constexpr int kSlots = SB_NSLOT;
constexpr int kWarp = 32;
constexpr int kMaxNodes = SB_MAX_NODES;
constexpr float kSentinel = 1.0e6f;  // reference's "unprofiled" runtime, PerformanceEvaluator.py:99

__device__ __forceinline__ float inf_f() { return __int_as_float(0x7f800000); }

// ---------------------------------------------------------------- the objective
// The fourteen scores the kernels compute, and the SB_FLAG_* bits that select each (sb_api.cu: decode_objective; every
// form also runs with SB_FLAG_RELEASE).  C is a job's completion, w its weight, d its due date, p its late penalty.
//   Obj               flags                                              score
//   Makespan          none                                               max C
//   TailMakespan      MAX_LATENESS                                       max (C + q), tails q = max d - d (L_max + max d)
//   Sum               SUM_COMPLETION                                     sum C
//   WeightedSum       SUM_COMPLETION | WEIGHTED                          sum w C
//   Tardiness         SUM_COMPLETION | DUE [| WEIGHTED]                  sum w max(C - d, 0), unit weights without WEIGHTED
//   LateCount         SUM_COMPLETION | DUE | LATE_COUNT [| WEIGHTED]     sum (C > d ? w : 0)
//   MaxTardiness      SUM_COMPLETION | DUE | MAX_TARDINESS [| WEIGHTED]  max w max(C - d, 0)
//   SquaredTardiness  SUM_COMPLETION | DUE | SQUARED [| WEIGHTED]        sum w max(C - d, 0)^2
//   LatePenalty       SUM_COMPLETION | DUE | LATE_PENALTY [| WEIGHTED]   sum (C > d ? p + w (C - d) : 0)
//   CompletionPenalty SUM_COMPLETION | DUE | COMPLETION_PENALTY [| WEIGHTED]
//                                                                        sum (w C + (C > d ? p : 0))
//   WorstMakespan     WORST_MAKESPAN                                     max_k M_k, M_k the makespan on scenario table k
//   MeanMakespan      MEAN_MAKESPAN                                      sum_k M_k, left fold in scenario order
//   WorstTardiness    SUM_COMPLETION | DUE | WORST_TARDINESS [| WEIGHTED] max_k S_k, S_k Tardiness's score on table k
//   MeanTardiness     SUM_COMPLETION | DUE | MEAN_TARDINESS [| WEIGHTED]  sum_k S_k, left fold in scenario order
// (the host runs the worst and mean completion time as these two with every due date +0: C >= +0, so the term
// w max(C - 0, 0) is w C bit for bit)
// Every other combination of those flags is refused.  The history of each form is in DESIGN.md.  New forms go at the
// end: a kernel's symbol holds its form's value.
enum class Obj {
  Makespan, TailMakespan, Sum, WeightedSum, Tardiness, LateCount, MaxTardiness, SquaredTardiness, LatePenalty,
  CompletionPenalty, WorstMakespan, MeanMakespan, WorstTardiness, MeanTardiness
};
// the score folds one score per scenario table (sb_set_scenarios): the makespans, or the total tardiness
__host__ __device__ constexpr bool obj_scenario(Obj o) {
  return o == Obj::WorstMakespan || o == Obj::MeanMakespan || o == Obj::WorstTardiness || o == Obj::MeanTardiness;
}
// the form ls_step folds inside one pass: the makespan or the tardiness for the scenario forms, the objective itself
// otherwise
__host__ __device__ constexpr Obj step_obj(Obj o) {
  return (o == Obj::WorstMakespan || o == Obj::MeanMakespan)     ? Obj::Makespan
         : (o == Obj::WorstTardiness || o == Obj::MeanTardiness) ? Obj::Tardiness
                                                                 : o;
}
// one scenario's score m folded into the score: an exact max (the worst forms), or a sum rounded at every add (the
// mean forms); both start at +0
template <Obj kObj>
__device__ __forceinline__ float scenario_fold(float score, float m) {
  return (kObj == Obj::WorstMakespan || kObj == Obj::WorstTardiness) ? fmaxf(score, m) : __fadd_rn(score, m);
}
// the score is a sum over the jobs, folded in schedule order
__host__ __device__ constexpr bool obj_sum(Obj o) {
  return o == Obj::Sum || o == Obj::WeightedSum || o == Obj::Tardiness || o == Obj::LateCount ||
         o == Obj::SquaredTardiness || o == Obj::LatePenalty || o == Obj::CompletionPenalty;
}
// the score reads the job weights (the caller's, or unit weights without SB_FLAG_WEIGHTED)
__host__ __device__ constexpr bool obj_weights(Obj o) {
  return o == Obj::WeightedSum || o == Obj::Tardiness || o == Obj::LateCount || o == Obj::MaxTardiness ||
         o == Obj::SquaredTardiness || o == Obj::LatePenalty || o == Obj::CompletionPenalty ||
         o == Obj::WorstTardiness || o == Obj::MeanTardiness;
}
// the score reads the due-date array: the due dates, or TailMakespan's tails
__host__ __device__ constexpr bool obj_due(Obj o) {
  return o == Obj::TailMakespan || o == Obj::Tardiness || o == Obj::LateCount || o == Obj::MaxTardiness ||
         o == Obj::SquaredTardiness || o == Obj::LatePenalty || o == Obj::CompletionPenalty ||
         o == Obj::WorstTardiness || o == Obj::MeanTardiness;
}
// the score reads the late-penalty array (sb_set_penalty)
__host__ __device__ constexpr bool obj_penalty(Obj o) {
  return o == Obj::LatePenalty || o == Obj::CompletionPenalty;
}

// ---------------------------------------------------------------- mbarrier + TMA bulk copy (1-D)
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
// thread-block cluster helpers (k_search_pos with the table split over a CTA pair)
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// every thread of every CTA of the cluster
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster window address of `addr` (a shared::cta address of this CTA) in the CTA with rank `rank`
__device__ __forceinline__ uint32_t cluster_map_shared(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  // make the inits visible to the async proxy (the TMA unit) before any bulk copy signals them
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a barrier that never completes is a bug (wrong byte count / misaligned copy);
// trap instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 26)) __trap();
  }
}
// global -> shared bulk copy through the TMA unit; completion is signalled on `bar` as `bytes`
// of transaction count.  dst, src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                             uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// named barriers (id 1..15; 0 is __syncthreads): `count` threads, a multiple of 32, take part in each phase.  Not the
// .aligned forms: a warp may reach them from inside a lane-divergent branch.
__device__ __forceinline__ void named_arrive(uint32_t id, uint32_t count) {
  asm volatile("barrier.cta.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void named_sync(uint32_t id, uint32_t count) {
  asm volatile("barrier.cta.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---------------------------------------------------------------- the list-scheduling step
// State: the 8 slot ready-times kept SORTED ascending in registers (f[0] <= ... <= f[7]).  Which
// physical slot holds which time does not influence any start time or the makespan (ties are
// between equal values), so the hot kernel evolves the sorted multiset only; the slot-exact
// variant lives in k_eval_full.
//
// A job with k = km1 + 1 GPUs starts at s = f[km1] (the k-th smallest), and the k smallest
// entries are replaced by v = s + hold.  With sh[i] = f[i + k] (+inf past the end) the new sorted
// state is  f'[i] = max(f[i], min(v, sh[i]))  — every surviving element below v moves down k
// places, the k copies of v follow, larger elements stay.  sh (and s, as element -1 of the same
// window) is produced by a 3-stage barrel shifter on the bits of km1: no dynamic register
// indexing, no divergence.
//
// Instruction mix: the step is bound by instruction issue, and before that by the ALU pipe, so work
// is spread over the ALU and FMA pipes at a low instruction count:
//   stage "by 4", lower half : 4 FSEL (ALU); predicates come from the bit inside the asm so that
//                              ptxas derives all three stage predicates with ONE R2P of the opt byte
//   stage "by 4", upper half : x = f + m with m = bit ? +inf : -0.0  (1 FSEL + 4 FADD, FMA pipe;
//                              f + -0.0 == f exactly, f + inf == inf) — doubles as the copy that
//                              keeps f intact for the final max
//   stages "by 2", "by 1"    : in-place predicated moves written as `@p mad.lo dst, src, one, 0`
//                              with `one` a run-time 1, so ptxas cannot fold them into SEL: they
//                              issue as predicated IMAD on the FMA pipe; +inf padding as predicated
//                              `add dst, dst, +inf`.  Ascending order reads only unmodified sources.
//   merge                    : 7 FMNMX (min) + 8 FMNMX (max) on the ALU pipe.
__device__ __forceinline__ void pmov_fma(float& dst, float src, int bit, int one) {
  int d = __float_as_int(dst);
  asm("{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %2, 0;\n\t@p mad.lo.s32 %0, %1, %3, 0;\n\t}"
      : "+r"(d)
      : "r"(__float_as_int(src)), "r"(bit), "r"(one));
  dst = __int_as_float(d);
}
// dst = +inf under the predicate, as `@p add.f32 dst, dst, +inf`: it depends on dst, so ptxas cannot
// hoist it into a SEL of a loop-invariant.
__device__ __forceinline__ void pinf_fma(float& dst, int bit) {
  asm("{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %1, 0;\n\t@p add.f32 %0, %0, 0f7F800000;\n\t}" : "+f"(dst) : "r"(bit));
}
// bit ? a : b with the predicate formed inside the asm (FSEL)
__device__ __forceinline__ float psel(float a, float b, int bit) {
  float r;
  asm("{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %3, 0;\n\tselp.f32 %0, %1, %2, p;\n\t}" : "=f"(r) : "f"(a), "f"(b), "r"(bit));
  return r;
}

// sm_90 has no 3-input max.f32, but it has the 3-input integer max (VIMNMX3).  The makespan fold only sees
// mk >= +0 and completions s + rt of non-negative runtimes: non-negative fp32 values order exactly like their bit
// patterns as signed integers, and a negative value (sign bit set) loses to mk either way.  One VIMNMX3 instead
// of two FMNMX, with the same result.
__device__ __forceinline__ float fmax3_mk(float mk, float b, float c) {
  return __int_as_float(__vimax3_s32(__float_as_int(mk), __float_as_int(b), __float_as_int(c)));
}

// The job's completion e = s + rt is folded into mk by the objective kObj; `w` is the job's weight, `d` its due date
// (TailMakespan: its tail q), `p` its late penalty, each read only by the forms that use it.  Every product and sum is
// rounded on its own (__fmul_rn, __fadd_rn: nvcc would otherwise contract them into one FFMA, which the oracle cannot
// reproduce).
//   Makespan     : only with kTrackMk (integer starts: the slot state holds s + ceil(rt), not the completion; several
//                  nodes: no single f[7] at the end), mk = max(mk, e).  `ph` pairs the completions of two consecutive
//                  steps into one 3-input max: 0 parks this step's completion in `pend`, 1 folds max(mk, pend, e);
//                  callers with unrolled loops pass t & 1 (a compile-time constant after unrolling), others pass -1
//                  for the plain 2-input max.  A parked value that is never folded is picked up by the final
//                  max(mk, pend) (LaneState::result).
//   TailMakespan : x = e + q, one rounding, folded like the makespan's completion (`ph`, `pend`) whatever kTrackMk
//                  says: f[7] is not x.  q = max_t d_t - d_j >= +0, so the score is L_max + max_t d_t >= +0.
//   the others   : mk is exact after every step (nothing parked, `ph` unused), one fold per step in schedule order,
//                  the oracle's left fold bit for bit.  Sum: mk + e.  WeightedSum: mk + w * e (w = 1 gives Sum bit for
//                  bit).  Tardiness: mk + w * max(e - d, +0) (d = 0 gives WeightedSum).  LateCount: mk + (e > d ? w :
//                  +0); a job that completes exactly at its due date is on time.  MaxTardiness: max(mk, w * max(e - d,
//                  +0)), Tardiness's term bit for bit folded with max; a job with no runtime (rt = +inf, w > 0) gives
//                  a +inf term.  SquaredTardiness: t = max(e - d, +0), Tardiness's term before the weight bit for
//                  bit, then mk + w * (t * t), three roundings; w = 1 gives the unweighted form bit for bit, and a
//                  job with no runtime a +inf term.  LatePenalty: x = e - d, then mk + (x > 0 ? p + w * x : +0), the
//                  product and the sum rounded on their own; p = +0 gives Tardiness's term bit for bit (+0 added to
//                  a positive finite value is exact), and a job with no runtime a +inf term.  CompletionPenalty:
//                  t = w * e, then t + p when e > d, then mk + t, each rounded on its own; p = +0 gives WeightedSum's
//                  term bit for bit (+0 added to a value >= +0 is exact), a job that completes exactly at its due date
//                  is on time, and a job with no runtime gives a +inf term.  k_eval_full folds this literal form.
// The slot update is the same under every objective: only the score differs.
// kRelease (SB_FLAG_RELEASE): the job starts no earlier than its release date `r`, s = max(f[km1], r) (ceil(r) under
// integer starts, made once by sb_set_release, so s stays an integer).  The slot update below stays valid because it
// only needs v >= f[km1]; r <= 0 gives s = f[km1] exactly.
template <bool kIntegerStarts, bool kTrackMk = kIntegerStarts, Obj kObj = Obj::Makespan, bool kRelease = false>
__device__ __forceinline__ void ls_step(float (&f)[8], float& mk, float& pend, float rt, int km1, int one, int ph,
                                        float w = 0.f, float d = 0.f, float r = 0.f, float p = 0.f) {
  const float INF = inf_f();
  const int b2 = km1 & 4, b1 = km1 & 2, b0 = km1 & 1;
  // stage "shift by 4"
  float x0 = psel(f[4], f[0], b2), x1 = psel(f[5], f[1], b2), x2 = psel(f[6], f[2], b2), x3 = psel(f[7], f[3], b2);
  const float m2 = psel(INF, -0.0f, b2);
  float x4 = f[4] + m2, x5 = f[5] + m2, x6 = f[6] + m2, x7 = f[7] + m2;
  // stage "shift by 2"
  pmov_fma(x0, x2, b1, one); pmov_fma(x1, x3, b1, one); pmov_fma(x2, x4, b1, one); pmov_fma(x3, x5, b1, one);
  pmov_fma(x4, x6, b1, one); pmov_fma(x5, x7, b1, one); pinf_fma(x6, b1); pinf_fma(x7, b1);
  // stage "shift by 1"
  pmov_fma(x0, x1, b0, one); pmov_fma(x1, x2, b0, one); pmov_fma(x2, x3, b0, one); pmov_fma(x3, x4, b0, one);
  pmov_fma(x4, x5, b0, one); pmov_fma(x5, x6, b0, one); pmov_fma(x6, x7, b0, one); pinf_fma(x7, b0);
  const float s = kRelease ? fmaxf(x0, r) : x0;  // = f[km1], or the release if later
  float v;
  if (kIntegerStarts) {
    // every entry of f is an integer here, so s is; the slot is usable again at s + ceil(rt)
    v = s + ceilf(rt);
  } else {
    v = s + rt;
  }
  if constexpr (kObj == Obj::TailMakespan) {
    const float x = __fadd_rn(kIntegerStarts ? s + rt : v, d);
    if (ph < 0) mk = fmaxf(mk, x);
    else if (ph == 0) pend = x;
    else mk = fmax3_mk(mk, pend, x);
  } else if constexpr (kObj != Obj::Makespan) {
    const float e = kIntegerStarts ? s + rt : v;
    // the late count: w * 1 = w and w * 0 = +0 exactly (w > 0 finite), so this adds (e > d ? w : +0); the product
    // keeps the tardiness form's data flow, which ptxas allocates without the spills a bare select causes in some
    // position-major search kernels at the 128-register cap
    if constexpr (kObj == Obj::LateCount) mk = __fadd_rn(mk, __fmul_rn(w, e > d ? 1.f : 0.f));
    // the maximum tardiness, max(mk, w * max(e - d, +0)), as one integer max over the product's bits: mk >= +0, and
    // w * (e - d) with w > 0 is either that term (e - d > 0), or +0, a negative value or -0 (e - d <= 0), which all
    // lose to mk as signed integers exactly as the +0 term does as a float.  Same value, one FMNMX fewer; the
    // float form gave two position-major search kernels more spills than their tardiness siblings
    else if constexpr (kObj == Obj::MaxTardiness)
      mk = __int_as_float(max(__float_as_int(mk), __float_as_int(__fmul_rn(w, __fsub_rn(e, d)))));
    else if constexpr (kObj == Obj::Tardiness) mk = __fadd_rn(mk, __fmul_rn(w, fmaxf(__fsub_rn(e, d), 0.f)));
    // the squared tardiness, mk + w * (t * t) with t = max(e - d, +0), as mk + w * (x * max(x, +0)) with x = e - d: for
    // x > 0 the same product, and for x <= 0 a +0 or -0 term, which adds to mk >= +0 exactly as the +0 term does.
    // Same value; the t * t form gave one position-major search kernel (PB 1, INT, a CTA-pair table, release dates)
    // 8 bytes of spills at the 128-register cap, where its tardiness sibling has none
    else if constexpr (kObj == Obj::SquaredTardiness) {
      const float x = __fsub_rn(e, d);
      mk = __fadd_rn(mk, __fmul_rn(w, __fmul_rn(x, fmaxf(x, 0.f))));
    }
    else if constexpr (kObj == Obj::LatePenalty) {
      const float x = __fsub_rn(e, d);
      mk = __fadd_rn(mk, x > 0.f ? __fadd_rn(p, __fmul_rn(w, x)) : 0.f);
    }
    // the completion penalty, t = w * e, then t + p when e > d, as t + (e > d ? p : +0): t >= +0, so adding +0 leaves
    // it exact.  Same value; the literal branch spilled 20 bytes in one multi-node search kernel, this form 4 to 8
    // bytes in ten single-node position-major search kernels (DESIGN §3.1, *Completion penalty*), all at 128 registers
    else if constexpr (kObj == Obj::CompletionPenalty)
      mk = __fadd_rn(mk, __fadd_rn(__fmul_rn(w, e), e > d ? p : 0.f));
    else if constexpr (kObj == Obj::WeightedSum) mk = __fadd_rn(mk, __fmul_rn(w, e));
    else mk = mk + e;
  } else if (kTrackMk) {
    const float e = kIntegerStarts ? s + rt : v;
    if (ph < 0) mk = fmaxf(mk, e);
    else if (ph == 0) pend = e;
    else mk = fmax3_mk(mk, pend, e);
  }
  f[0] = fmaxf(f[0], fminf(v, x1));
  f[1] = fmaxf(f[1], fminf(v, x2));
  f[2] = fmaxf(f[2], fminf(v, x3));
  f[3] = fmaxf(f[3], fminf(v, x4));
  f[4] = fmaxf(f[4], fminf(v, x5));
  f[5] = fmaxf(f[5], fminf(v, x6));
  f[6] = fmaxf(f[6], fminf(v, x7));
  f[7] = fmaxf(f[7], v);
}

__device__ __forceinline__ unsigned long long pack_key(float mk, uint32_t id) {
  return (static_cast<unsigned long long>(__float_as_uint(mk)) << 32) | id;
}

// counter-based RNG: one 64-bit mix per draw, keyed by (seed, stream id, counter)
__device__ __host__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9e3779b97f4a7c15ull;
  z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
  z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
  return z ^ (z >> 31);
}
__device__ __host__ __forceinline__ uint64_t rng_u64(uint64_t seed, uint64_t stream, uint64_t ctr) {
  return mix64(mix64(seed ^ (stream * 0xd1342543de82ef95ull)) + ctr * 0x2545f4914f6cdd1dull);
}

}  // namespace sb
