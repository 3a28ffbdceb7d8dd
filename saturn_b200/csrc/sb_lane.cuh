// sb_lane.cuh — per-lane evaluation state and the helpers shared by the evaluation kernel (sb_eval.cu)
// and the large-J fused search kernel (sb_search.cu).
#pragma once
#include "sb_internal.h"

namespace sb {

struct PrioChunk {
  uint32_t w[8];  // 32 bytes = 32 (u8) or 16 (u16) schedule positions
};
// kReadOnly: the rows are not written during the kernel (evaluation) -> non-coherent path; the fused
// search round writes accepted moves back into the same rows, so it uses the coherent form.
// sm_90 has no 256-bit global load: the 32-byte chunk (p 32-byte aligned, one sector) is two 128-bit loads.
template <bool kReadOnly>
__device__ __forceinline__ PrioChunk ld_prio32(const uint8_t* p) {
  PrioChunk c;
  if (kReadOnly) {
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                 "ld.global.nc.L1::no_allocate.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(c.w[0]), "=r"(c.w[1]), "=r"(c.w[2]), "=r"(c.w[3]), "=r"(c.w[4]), "=r"(c.w[5]), "=r"(c.w[6]),
                   "=r"(c.w[7])
                 : "l"(p));
  } else {
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
                 "ld.global.L1::no_allocate.v4.u32 {%4,%5,%6,%7}, [%8+16];"
                 : "=r"(c.w[0]), "=r"(c.w[1]), "=r"(c.w[2]), "=r"(c.w[3]), "=r"(c.w[4]), "=r"(c.w[5]), "=r"(c.w[6]),
                   "=r"(c.w[7])
                 : "l"(p)
                 : "memory");
  }
  return c;
}

// The per-job fp32 arrays a kernel stages beside its table, in this order: the weights (obj_weights), the due dates or
// tails (obj_due), the release dates (SB_FLAG_RELEASE), the late penalties (obj_penalty).  Each is padded to 16 bytes
// (each kernel spells the padding out per array: computing it once changes the generated code) and is fetched by
// stage_job_array with TMA bulk copies in the table's mbarrier phase.
__device__ __forceinline__ void stage_job_array(uint8_t* dst, const float* src, uint32_t bytes, uint64_t* bar) {
  const uint8_t* s = reinterpret_cast<const uint8_t*>(src);
  for (uint32_t off = 0; off < bytes; off += 32768u) tma_bulk_g2s(dst + off, s + off, min(32768u, bytes - off), bar);
}

// Per-lane evaluation state + the per-job step.
// ADDR = 1 (shared-memory table and opt rows only): the two look-up addresses of a step are formed with
// `mad.lo` on run-time multipliers, which ptxas must issue as IMAD on the FMA pipe instead of IADD3 / LEA on
// the ALU pipe — the step is bound by the ALU pipe (half rate) and by issue together, so the same instruction
// count with two fewer ALU instructions is the cheaper mix.
// OBJ: the objective that ls_step folds (sb_common.cuh).  REL (SB_FLAG_RELEASE, with any objective): no job starts
// before its release date.  HOME: where the per-job arrays these read live (stage_job_array) — 1: in shared memory
// beside the table, 2: in global memory, read with ld.global.nc.
template <bool INT, bool MULTI, int ADDR = 0, Obj OBJ = Obj::Makespan, int HOME = 0, bool REL = false>
struct LaneState {
  static constexpr bool kW = obj_weights(OBJ), kD = obj_due(OBJ), kP = obj_penalty(OBJ);
  float f[8];
  float mk;
  float pend;  // a completion time parked by an even step (see ls_step; the makespan forms only)
  const uint8_t* orow;  // this candidate's opt bytes (shared memory or global)
  const float* tab;     // runtime table (shared memory or global)
  const float* wt;      // kW: the job weights [J]
  const float* dd;      // kD: the job due dates [J] (or delivery tails)
  const float* rr;      // REL: the job release dates [J]
  const float* pp;      // kP: the job late penalties [J]
  int SG;
  int one;
  uint32_t orow_s, tab_s, four;  // ADDR = 1: shared-window addresses of orow / tab, and a run-time 4
  uint32_t wt_s, dd_s, rr_s, pp_s;  // ADDR = 1: shared-window addresses of wt / dd / rr / pp
  float4* ns;  // MULTI: lane-private node-state column; node n lives at ns[(2n)*32], ns[(2n+1)*32]
  int cur;     // MULTI: the node whose state is currently in f[] (its shared-memory copy is stale)

  __device__ __forceinline__ void reset(int nodes) {
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = 0.f;
    mk = 0.f;
    pend = 0.f;
    cur = 0;
    if (MULTI) {
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int n = 0; n < 2 * nodes; ++n) ns[n * 32] = z;
    }
  }
  // MULTI: bring node n's sorted state into the registers (write the previous node's back first).
  // Lanes whose job stays on the same node as their previous job skip the shared-memory round trip.
  __device__ __forceinline__ void switch_node(int n) {
    if (n != cur) {
      float4* old = ns + (2 * cur) * 32;
      old[0] = make_float4(f[0], f[1], f[2], f[3]);
      old[32] = make_float4(f[4], f[5], f[6], f[7]);
      const float4* slot = ns + (2 * n) * 32;
      const float4 lo = slot[0], hi = slot[32];
      f[0] = lo.x; f[1] = lo.y; f[2] = lo.z; f[3] = lo.w;
      f[4] = hi.x; f[5] = hi.y; f[6] = hi.z; f[7] = hi.w;
      cur = n;
    }
  }
  // the two look-ups of a step (opt byte, then runtime) do not depend on the slot state, so callers
  // that read from global memory resolve a batch of positions first (memory-level parallelism)
  __device__ __forceinline__ int lookup_opt(int j) const { return orow[j]; }
  __device__ __forceinline__ float lookup_rt(int j, int o) const {
    return MULTI ? tab[j * 8 + (o & 7)] : tab[j * SG + o];
  }
  // the job's entry of a per-job array: shared memory (HOME = 1) or global memory (HOME = 2)
  __device__ __forceinline__ float job_at(const float* a, int j) const { return HOME == 1 ? a[j] : __ldg(a + j); }
  // the job's weight, due date (or tail), release date and late penalty; 0 where the kernel reads none
  __device__ __forceinline__ float lookup_w(int j) const { if constexpr (kW) return job_at(wt, j); else return 0.f; }
  __device__ __forceinline__ float lookup_d(int j) const { if constexpr (kD) return job_at(dd, j); else return 0.f; }
  __device__ __forceinline__ float lookup_r(int j) const { if constexpr (REL) return job_at(rr, j); else return 0.f; }
  __device__ __forceinline__ float lookup_p(int j) const { if constexpr (kP) return job_at(pp, j); else return 0.f; }
  // ph: t & 1 inside fully unrolled loops, -1 elsewhere (see ls_step); w, d, r, p: the job's weight, due date (or
  // tail), release date and late penalty, each read only where the objective (or REL) uses it
  __device__ __forceinline__ void step_resolved(int o, float rt, int ph = -1, float w = 0.f, float d = 0.f,
                                                float r = 0.f, float p = 0.f) {
    if (!MULTI) {
      ls_step<INT, INT, OBJ, REL>(f, mk, pend, rt, o & 7, one, ph, w, d, r, p);
    } else {
      switch_node(o >> 3);
      ls_step<INT, true, OBJ, REL>(f, mk, pend, rt, o & 7, one, ph, w, d, r, p);
    }
  }
  // ADDR = 1: the two look-ups as separate gathers, so that the streamed loop of k_eval_tiles can issue a whole
  // batch of opt-byte gathers, then the batch's runtime gathers, ahead of the steps that consume them
  __device__ __forceinline__ uint32_t gather_opt(int j) const {
    uint32_t oa, o;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(oa) : "r"(j), "r"(one), "r"(orow_s));
    asm("ld.shared.u8 %0, [%1];" : "=r"(o) : "r"(oa));
    return o;
  }
  __device__ __forceinline__ float gather_rt(int j, uint32_t o) const {
    uint32_t idx, ta;
    float rt;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(idx) : "r"(j), "r"(SG), "r"(o));
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(ta) : "r"(idx), "r"(four), "r"(tab_s));
    asm("ld.shared.f32 %0, [%1];" : "=f"(rt) : "r"(ta));
    return rt;
  }
  // ADDR = 1: the job's entry of a per-job array at shared-window address `base`, its address formed on the FMA pipe
  // like the two above
  __device__ __forceinline__ float gather_at(uint32_t base, int j) const {
    uint32_t a;
    float v;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(a) : "r"(j), "r"(four), "r"(base));
    asm("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
    return v;
  }
  __device__ __forceinline__ float gather_w(int j) const { if constexpr (kW) return gather_at(wt_s, j); else return 0.f; }
  __device__ __forceinline__ float gather_d(int j) const { if constexpr (kD) return gather_at(dd_s, j); else return 0.f; }
  __device__ __forceinline__ float gather_r(int j) const { if constexpr (REL) return gather_at(rr_s, j); else return 0.f; }
  __device__ __forceinline__ float gather_p(int j) const { if constexpr (kP) return gather_at(pp_s, j); else return 0.f; }
  __device__ __forceinline__ void step(int j, int ph = -1) {
    if (!MULTI && ADDR == 1) {
      const uint32_t o = gather_opt(j);
      ls_step<INT, INT, OBJ, REL>(f, mk, pend, gather_rt(j, o), static_cast<int>(o & 7u), one, ph, gather_w(j),
                                  gather_d(j), gather_r(j), gather_p(j));
      return;
    }
    const int o = orow[j];
    if (!MULTI) {
      const float rt = tab[j * SG + o];
      ls_step<INT, INT, OBJ, REL>(f, mk, pend, rt, o & 7, one, ph, lookup_w(j), lookup_d(j), lookup_r(j),
                                  lookup_p(j));
    } else {
      const int col = o & 7;  // reduced table only: opt = (node << 3) | (k - 1)
      const float rt = tab[j * 8 + col];
      switch_node(o >> 3);
      ls_step<INT, true, OBJ, REL>(f, mk, pend, rt, col, one, ph, lookup_w(j), lookup_d(j), lookup_r(j),
                                   lookup_p(j));
    }
  }
  // the tail makespan is tracked in mk at every shape: f[7] is a completion, not a tail sum.
  // LateCount: a job with no runtime (+inf cell) adds only its weight to the count, but the candidate is infeasible
  // and scores +inf, as under every other objective.  Such a job leaves +inf in the slots it held, and slot times never
  // decrease, so one look at each node's latest slot time at the end finds it (`nodes`: MULTI only; the node in
  // f[] is checked there, the others in their shared-memory columns, where a stale copy of it is never +inf wrongly).
  __device__ __forceinline__ float result(int nodes = 1) const {
    if constexpr (OBJ == Obj::LateCount) {
      float last = f[7];
      if constexpr (MULTI)
        for (int n = 0; n < nodes; ++n) last = fmaxf(last, ns[(2 * n + 1) * 32].w);
      return last == inf_f() ? inf_f() : mk;
    }
    if constexpr (OBJ == Obj::Makespan) return (INT || MULTI) ? fmaxf(mk, pend) : f[7];
    else if constexpr (OBJ == Obj::TailMakespan) return fmaxf(mk, pend);
    else return mk;
  }
  // the running score a snapshot of the incremental rounds stores (SearchFuse::snap): only the makespan forms park a
  // completion, so the other objectives' snapshots are exact at any step, not only after an even number of steps
  __device__ __forceinline__ float running() const {
    return (OBJ == Obj::Makespan || OBJ == Obj::TailMakespan) ? fmaxf(mk, pend) : mk;
  }
};

template <int PB>
__device__ __forceinline__ int prio_at(const uint32_t* w, int t) {
  // one PRMT per position: pick byte(s) t of the word, zero the rest (selector nibble 4 = byte 0 of
  // the second operand, which is 0)
  if (PB == 1) return static_cast<int>(__byte_perm(w[t >> 2], 0u, 0x4440u + (t & 3)));
  return static_cast<int>(__byte_perm(w[t >> 1], 0u, (t & 1) ? 0x4432u : 0x4410u));
}

// Returns true in the one lane whose candidate lowered *best_key (false everywhere else).
__device__ __forceinline__ bool fold_best(unsigned long long* best_key, bool active, float mk, uint32_t id, int lane) {
  const uint32_t bits = active ? __float_as_uint(mk) : 0xffffffffu;
  const uint32_t mn = __reduce_min_sync(0xffffffffu, bits);
  const uint32_t who = __ballot_sync(0xffffffffu, bits == mn);
  bool lowered = false;
  if (lane == __ffs(who) - 1 && active) {
    const unsigned long long key = pack_key(mk, id);
    if (key < *reinterpret_cast<volatile unsigned long long*>(best_key)) lowered = key < atomicMin(best_key, key);
  }
  return lowered;
}

// Which chains stop moving inside a multi-round launch.  The tail below saves the rows of the chain that holds
// the population's best key, so those rows must still be the candidate the key was scored on: a chain whose
// candidate is strictly better than the incumbent saved BEFORE this launch (keys[1]; only the tail of a launch
// writes it, after every CTA has finished) stops moving for the rest of the launch.  The rule reads nothing that
// other warps write during the launch, so a search is reproducible bit for bit whatever the interleaving of
// warps (the first version froze the chain that won the atomicMin race, which made runs depend on timing).
__device__ __forceinline__ uint32_t launch_incumbent_bits(const SearchFuse& sf) {
  return sf.keep.keys != nullptr
             ? static_cast<uint32_t>(*reinterpret_cast<volatile unsigned long long*>(sf.keep.keys + 1) >> 32)
             : 0u;
}

// Tail of a fused search round: every thread's accepted row bytes are fenced, the CTA that finishes last
// has therefore seen the whole round; its first warp saves the incumbent's rows if keys[0] improved on
// keys[1] (what k_keep_best does as a separate launch for the unfused rounds).
__device__ __forceinline__ void keep_best_tail(const SearchFuse& sf) {
  __threadfence();
  __syncthreads();
  int mine = 0;
  if (threadIdx.x == 0) {
    const unsigned done = atomicAdd(sf.keep.counter, 1u);
    mine = done == gridDim.x - 1;
    if (mine) *sf.keep.counter = 0;
  }
  if (!__syncthreads_or(mine) || threadIdx.x >= 32) return;
  __threadfence();
  const int lane = threadIdx.x;
  const unsigned long long key = *reinterpret_cast<volatile unsigned long long*>(sf.keep.keys);
  const unsigned long long saved = *reinterpret_cast<volatile unsigned long long*>(sf.keep.keys + 1);
  // only a strictly better MAKESPAN replaces the saved incumbent: exactly the chains that froze (frozen_by).  A
  // lower key with the saved score (a lower chain id) names a chain that kept moving, so its rows are no longer the
  // ones that key was scored on: the best key goes back to the saved incumbent's, or the next k_keep_best (an
  // injection, an unfused round) would save that chain's current rows under it.
  if ((key >> 32) >= (saved >> 32)) {
    if (lane == 0 && key != saved) sf.keep.keys[0] = saved;
    return;
  }
  const long long c = static_cast<long long>(((key & 0xffffffffull) - (sf.chain_base & 0xffffffffull)) & 0xffffffffull);
  if (c >= sf.keep.chains) return;
  const uint4* so = reinterpret_cast<const uint4*>(sf.cur_o + c * sf.keep.stride_o);
  const uint4* sp = reinterpret_cast<const uint4*>(sf.cur_p + c * sf.keep.stride_p);
  for (int i = lane; i * 16 < sf.keep.stride_o; i += 32) reinterpret_cast<uint4*>(sf.keep.best_o)[i] = __ldcg(so + i);
  for (int i = lane; i * 16 < sf.keep.stride_p; i += 32) reinterpret_cast<uint4*>(sf.keep.best_p)[i] = __ldcg(sp + i);
  __syncwarp();
  if (lane == 0) sf.keep.keys[1] = key;
}

// ---- SEARCH variant: one Metropolis round fused into the tile kernel.  The rows a warp fetched
// are the chains' CURRENT candidates; every lane applies its own random move to its private
// shared-memory rows, scores the result, decides acceptance and — only when accepted — writes the
// few changed bytes back to the chain's rows in HBM.  No proposal buffer, no separate propose /
// accept kernels (the bulk of an unfused round's traffic).
struct Move {
  int kind;  // 0 none, 1 opt byte of job a changed, 2 positions a,b swapped, 3 positions [a..b] rewritten
  int a, b;
  int va, vb;  // kind 1: va = the previous opt byte; kind 2: the jobs that were at positions a and b;
               // kind 3: the job travelled from position va to position vb
};

__device__ __forceinline__ uint32_t bounded32(uint64_t r, uint32_t n) {
  return static_cast<uint32_t>((static_cast<uint64_t>(static_cast<uint32_t>(r >> 32)) * n) >> 32);
}

template <int PB>
__device__ __forceinline__ int smem_prio_ld(const uint8_t* row, int i) {
  return PB == 1 ? row[i] : reinterpret_cast<const uint16_t*>(row)[i];
}
template <int PB>
__device__ __forceinline__ void smem_prio_st(uint8_t* row, int i, int v) {
  if (PB == 1) row[i] = static_cast<uint8_t>(v);
  else reinterpret_cast<uint16_t*>(row)[i] = static_cast<uint16_t>(v);
}

// `orow` / `prow` are the lane's rows in SHARED memory: the move is applied in place.
template <int PB>
__device__ __forceinline__ Move apply_move(const SearchFuse& sf, int round, int J, uint64_t gid, uint8_t* orow,
                                           uint8_t* prow) {
  Move m;
  m.kind = 0; m.a = 0; m.b = 0; m.va = 0; m.vb = 0;
  const uint64_t r0 = rng_u64(sf.seed, gid, 4ull * round + 0);
  const uint64_t r1 = rng_u64(sf.seed, gid, 4ull * round + 1);
  const uint64_t r2 = rng_u64(sf.seed, gid, 4ull * round + 2);
  const uint32_t kind = bounded32(r0, 100);
  if (sf.nodes > 1 && kind >= 85) {  // move one job to another node (milp.py:117-137)
    const int j = bounded32(r1, J);
    const uint8_t curv = orow[j];
    int nn = bounded32(r2, sf.nodes - 1);
    if (nn >= (curv >> 3)) ++nn;
    orow[j] = static_cast<uint8_t>((curv & 7) | (nn << 3));
    m.kind = 1; m.a = j; m.va = curv;
    return m;
  }
  if (kind < 30) {  // change one job's option (keeping its node)
    const int j = bounded32(r1, J);
    const int n = sf.nvalid[j];
    if (n > 1) {
      const int pick = bounded32(r2, n - 1);
      const uint8_t curv = orow[j];
      const uint8_t node_bits = sf.nodes > 1 ? (curv & 0xf8) : 0;
      const uint8_t cur_opt = sf.nodes > 1 ? (curv & 7) : curv;
      uint8_t nv = sf.vopt[j * kSlots + pick];
      if (nv == cur_opt) nv = sf.vopt[j * kSlots + n - 1];
      orow[j] = nv | node_bits;
      m.kind = 1; m.a = j; m.va = curv;
      return m;
    }
  }
  if (J < 2) return m;
  const int a = bounded32(r1, J);
  if (kind < 70) {  // swap two priorities
    int b = bounded32(r2, J - 1);
    if (b >= a) ++b;
    const int va = smem_prio_ld<PB>(prow, a), vb = smem_prio_ld<PB>(prow, b);
    smem_prio_st<PB>(prow, a, vb);
    smem_prio_st<PB>(prow, b, va);
    m.kind = 2; m.a = a; m.b = b; m.va = va; m.vb = vb;
    return m;
  }
  // re-insert the job at position a up to 48 places earlier or later
  const int span = J - 1 < 48 ? J - 1 : 48;
  int d = 1 + static_cast<int>(bounded32(r2, 2 * span));  // 1..2*span
  int b = d <= span ? a + d : a - (d - span);
  if (b < 0) b = 0;
  if (b > J - 1) b = J - 1;
  if (b == a) return m;
  const int va = smem_prio_ld<PB>(prow, a);
  if (a < b) {
    for (int i = a; i < b; ++i) smem_prio_st<PB>(prow, i, smem_prio_ld<PB>(prow, i + 1));
  } else {
    for (int i = a; i > b; --i) smem_prio_st<PB>(prow, i, smem_prio_ld<PB>(prow, i - 1));
  }
  smem_prio_st<PB>(prow, b, va);
  m.kind = 3; m.a = a < b ? a : b; m.b = a < b ? b : a; m.va = a; m.vb = b;
  return m;
}

// The window of a round, from one 64-bit draw shared by the warp.  bias 0: uniform over the nwin windows.
// bias 1 (experiment, test hook HOOK_WINDOW_BIAS): P(w) proportional to w + 1 — later windows skip more
// of the schedule (mean resume point 0.58 instead of 0.44 of the way in at 8 windows) at the price of fewer
// moves near the front of the schedule.
__device__ __forceinline__ int draw_window(uint64_t r, int nwin, int bias) {
  if (bias == 0) return static_cast<int>(bounded32(r, nwin));
  // triangular: pick t uniform in [0, nwin (nwin + 1) / 2) and invert the cumulative sum
  const uint32_t tot = static_cast<uint32_t>(nwin) * (nwin + 1) / 2;
  const uint32_t t = bounded32(r, tot);
  int w = static_cast<int>((sqrtf(8.f * static_cast<float>(t) + 1.f) - 1.f) * 0.5f);
  while (static_cast<uint32_t>(w + 1) * (w + 2) / 2 <= t) ++w;   // fix the float rounding
  while (static_cast<uint32_t>(w) * (w + 1) / 2 > t) --w;
  return w;
}

// Windowed form of apply_move (incremental rounds, see SearchFuse::snap): the first schedule position a move
// changes lies inside [w0, w0 + wlen), positions before w0 are untouched.  Same move kinds and mix; a job is
// addressed through its position (the option of the job scheduled i-th changes), a swap pairs a position of the
// window with any later-or-equal position, a re-insertion moves a job forward from the window or back into it.
template <int PB>
__device__ __forceinline__ Move apply_move_win(const SearchFuse& sf, int round, int J, uint64_t gid, uint8_t* orow,
                                               uint8_t* prow, int w0, int wlen) {
  Move m;
  m.kind = 0; m.a = 0; m.b = 0; m.va = 0; m.vb = 0;
  const uint64_t r0 = rng_u64(sf.seed, gid, 4ull * round + 0);
  const uint64_t r1 = rng_u64(sf.seed, gid, 4ull * round + 1);
  const uint64_t r2 = rng_u64(sf.seed, gid, 4ull * round + 2);
  const uint32_t kind = bounded32(r0, 100);
  const int a = w0 + static_cast<int>(bounded32(r1, wlen));
  if (kind < 30) {  // change the option of the job scheduled a-th
    const int j = smem_prio_ld<PB>(prow, a);
    const int n = sf.nvalid[j];
    if (n > 1) {
      const int pick = bounded32(r2, n - 1);
      const uint8_t curv = orow[j];
      uint8_t nv = sf.vopt[j * kSlots + pick];
      if (nv == curv) nv = sf.vopt[j * kSlots + n - 1];
      orow[j] = nv;
      m.kind = 1; m.a = j; m.va = curv;
      return m;
    }
  }
  const int tail = J - w0;  // positions from the window's start on
  if (tail < 2) return m;
  if (kind < 70) {  // swap position a with another position >= w0
    int b = w0 + static_cast<int>(bounded32(r2, tail - 1));
    if (b >= a) ++b;
    const int va = smem_prio_ld<PB>(prow, a), vb = smem_prio_ld<PB>(prow, b);
    smem_prio_st<PB>(prow, a, vb);
    smem_prio_st<PB>(prow, b, va);
    m.kind = 2; m.a = a; m.b = b; m.va = va; m.vb = vb;
    return m;
  }
  // re-insertion over up to 48 places: the job at a moves later, or a job from later moves to a
  const int span = J - 1 < 48 ? J - 1 : 48;
  const uint32_t dd = bounded32(r2, 2 * span);
  int b = a + 1 + static_cast<int>(dd >> 1);
  if (b > J - 1) b = J - 1;
  if (b == a) return m;
  if (dd & 1) {  // a -> b
    const int va = smem_prio_ld<PB>(prow, a);
    for (int i = a; i < b; ++i) smem_prio_st<PB>(prow, i, smem_prio_ld<PB>(prow, i + 1));
    smem_prio_st<PB>(prow, b, va);
    m.va = a; m.vb = b;
  } else {  // b -> a
    const int vb = smem_prio_ld<PB>(prow, b);
    for (int i = b; i > a; --i) smem_prio_st<PB>(prow, i, smem_prio_ld<PB>(prow, i - 1));
    smem_prio_st<PB>(prow, a, vb);
    m.va = b; m.vb = a;
  }
  m.kind = 3; m.a = a; m.b = b;
  return m;
}

// A rejected move is taken back so that the rows in shared memory stay the chain's current candidate
// (several rounds run on the same tile, see k_eval_tiles).
template <int PB>
__device__ __forceinline__ void undo_move(const Move& m, uint8_t* orow, uint8_t* prow) {
  if (m.kind == 1) {
    orow[m.a] = static_cast<uint8_t>(m.va);
  } else if (m.kind == 2) {
    smem_prio_st<PB>(prow, m.a, m.va);
    smem_prio_st<PB>(prow, m.b, m.vb);
  } else if (m.kind == 3) {
    const int from = m.vb, to = m.va;  // the job sits at `from` and goes back to `to`
    const int job = smem_prio_ld<PB>(prow, from);
    if (from < to) {
      for (int i = from; i < to; ++i) smem_prio_st<PB>(prow, i, smem_prio_ld<PB>(prow, i + 1));
    } else {
      for (int i = from; i > to; --i) smem_prio_st<PB>(prow, i, smem_prio_ld<PB>(prow, i - 1));
    }
    smem_prio_st<PB>(prow, to, job);
  }
}

template <int PB>
__device__ __forceinline__ void write_back(const Move& m, const uint8_t* orow, const uint8_t* prow, uint8_t* go,
                                           uint8_t* gp) {
  if (m.kind == 1) {
    go[m.a] = orow[m.a];
  } else if (m.kind == 2) {
    // positions a and b exchange their jobs (values carried in the move)
    if (PB == 1) { gp[m.a] = static_cast<uint8_t>(m.vb); gp[m.b] = static_cast<uint8_t>(m.va); }
    else {
      reinterpret_cast<uint16_t*>(gp)[m.a] = static_cast<uint16_t>(m.vb);
      reinterpret_cast<uint16_t*>(gp)[m.b] = static_cast<uint16_t>(m.va);
    }
  } else if (m.kind == 3) {
    for (int i = m.a; i <= m.b; ++i) {
      if (PB == 1) gp[i] = prow[i];
      else reinterpret_cast<uint16_t*>(gp)[i] = reinterpret_cast<const uint16_t*>(prow)[i];
    }
  }
}

// Streamed rows (position-major search, sb_search.cu): overwrite position `pos` with `val` in the 256-bit chunk `c` held in
// registers (no dynamic register indexing: the word is selected by predication over the 8 words).
template <int PB>
__device__ __forceinline__ void patch_chunk(PrioChunk& q, int c, int pos, int val) {
  constexpr int STEPS = 32 / PB;
  if (pos / STEPS != c) return;
  const int t = pos % STEPS;
  const int widx = PB == 1 ? (t >> 2) : (t >> 1);
  const int sh = PB == 1 ? (t & 3) * 8 : (t & 1) * 16;
  const uint32_t mask = (PB == 1 ? 0xffu : 0xffffu) << sh;
  const uint32_t ins = static_cast<uint32_t>(val) << sh;
#pragma unroll
  for (int i = 0; i < 8; ++i)
    if (i == widx) q.w[i] = (q.w[i] & ~mask) | ins;
}

}  // namespace sb
