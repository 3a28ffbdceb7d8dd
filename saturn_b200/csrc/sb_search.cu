// sb_search.cu — the search that replaces `prob.solve(solver)` (saturn/solver/milp.py:321-327).
//
// The reference minimises makespan by branch-and-bound over the MILP of milp.py:96-319 with a
// wall-clock limit and a warm start (milp.py:103-104,151-155,197-202,323-325).  Here a population
// of candidates (one per "chain") lives in HBM and each round does, entirely on the device:
//   propose  : apply one move to the chain's current candidate (swap two priorities / re-insert a
//              job elsewhere in the order / change one job's option / move it to another node);
//   evaluate : the list-scheduling step of sb_eval.cu (the measured hot path), folding
//              (makespan, global chain id) into a 64-bit arg-min key;
//   keep     : if the key improved, save that candidate's encoding as the incumbent;
//   accept   : Metropolis rule per chain at the round's temperature.
// Where the rows fit in shared memory all four happen inside k_eval_tiles<..., SEARCH> (sb_eval.cu), up
// to 8 rounds per launch, tournament resampling included.  This file holds the rest: population
// initialisation, injection, the copy-kernel form of the tournament, the position-major round kernel
// for large J (k_search_pos) and the unfused propose / keep / accept kernels (fallback and cross-check).
// Random numbers are counter-based (seed, global chain id, round), so a run is reproducible and
// independent of how chains are sharded across GPUs.
#include "sb_search.h"
#include "sb_lane.cuh"

namespace sb {

__device__ __forceinline__ uint32_t bounded(uint64_t r, uint32_t n) {  // uniform in [0, n)
  return static_cast<uint32_t>((static_cast<uint64_t>(static_cast<uint32_t>(r >> 32)) * n) >> 32);
}

template <int PB>
__device__ __forceinline__ int prio_ld(const uint8_t* row, int i) {
  return PB == 1 ? row[i] : reinterpret_cast<const uint16_t*>(row)[i];
}
template <int PB>
__device__ __forceinline__ void prio_st(uint8_t* row, int i, int v) {
  if (PB == 1) row[i] = static_cast<uint8_t>(v);
  else reinterpret_cast<uint16_t*>(row)[i] = static_cast<uint16_t>(v);
}

// ---- initial population: random valid options, random permutation (Fisher-Yates); thread per chain
template <int PB>
__global__ void k_init_population(SearchDev s) {
  const long long c = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (c >= s.chains) return;
  uint8_t* orow = s.cur_o + c * s.stride_o;
  uint8_t* prow = s.cur_p + c * s.stride_p;
  const uint64_t gid = s.chain_base + static_cast<uint64_t>(c);
  for (int j = 0; j < s.J; ++j) {
    const uint64_t r = rng_u64(s.seed, gid, 0x100000000ull + j);
    uint8_t ob = s.vopt[j * kSlots + bounded(r, s.nvalid[j])];
    if (s.nodes > 1) ob = static_cast<uint8_t>((ob & 7) | (bounded(rng_u64(s.seed, gid, 0x300000000ull + j), s.nodes) << 3));
    orow[j] = ob;
    prio_st<PB>(prow, j, j);
  }
  for (int i = s.J - 1; i > 0; --i) {
    const uint64_t r = rng_u64(s.seed, gid, 0x200000000ull + i);
    const int k = bounded(r, i + 1);
    const int a = prio_ld<PB>(prow, i), b = prio_ld<PB>(prow, k);
    prio_st<PB>(prow, i, b);
    prio_st<PB>(prow, k, a);
  }
}

// ---- initial population, built in SHARED memory: one thread per chain shuffles its priority row there
// (the Fisher-Yates swaps are dependent random accesses: a shared-memory access each instead of the
// global-memory round trip of the serial per-thread version above), then the CTA writes the finished rows out with coalesced 32-bit stores
// (padding included, so the rows need no memset).  The shuffle draws from a per-chain 32-bit LCG seeded by the
// counter-based generator (one IMAD per draw on the serial path instead of two 64-bit mixes); the option
// bytes are independent of each other, so they are not staged at all: the write-out derives the four bytes of a
// word from two 32-bit hashes of (chain id, word) (16 random bits per byte; at most 64 options per job, bias
// < 1e-3), for the job or — POS, opt bytes in schedule order — for the jobs at those four positions, with the
// (row, word) pairs of the CTA dealt over all threads and the option lists staged in shared memory.  Only the
// priority rows and those lists live in shared memory: 24 warps per SM at J = 256.
// 32-bit avalanche (murmur3 finaliser): the option choices of a word need 4 x 16 random bits per (chain, word)
__device__ __forceinline__ uint32_t hash32(uint32_t h) {
  h ^= h >> 16; h *= 0x85ebca6bu; h ^= h >> 13; h *= 0xc2b2ae35u; h ^= h >> 16;
  return h;
}

template <int PB, bool POS>
__global__ void k_init_population_smem(SearchDev s, int row_p) {
  extern __shared__ __align__(16) uint8_t sm_rows[];
  const int T = blockDim.x;
  const int J = s.J;
  uint8_t* sp = sm_rows + static_cast<size_t>(threadIdx.x) * row_p;
  // the proposable-option lists of all jobs, staged once per CTA: [J][8] opt bytes + [J] counts
  uint8_t* vopt_s = sm_rows + static_cast<size_t>(T) * row_p;
  uint8_t* nval_s = vopt_s + static_cast<size_t>(J) * kSlots;
  for (int x = threadIdx.x; x < J * kSlots; x += T) vopt_s[x] = s.vopt[x];
  for (int x = threadIdx.x; x < J; x += T) nval_s[x] = static_cast<uint8_t>(s.nvalid[x]);
  const long long c0 = static_cast<long long>(blockIdx.x) * T;
  const long long c = c0 + threadIdx.x;
  if (c < s.chains) {
    const uint64_t gid = s.chain_base + static_cast<uint64_t>(c);
    for (int x = J * PB; x < row_p; ++x) sp[x] = 0;
    for (int j = 0; j < J; ++j) prio_st<PB>(sp, j, j);
    // Fisher-Yates on a per-chain 32-bit LCG seeded by the counter-based generator: one IMAD per draw on the
    // serial path, the bounded index from the HIGH bits (mulhi)
    uint32_t x = static_cast<uint32_t>(rng_u64(s.seed, gid, 0x200000000ull) >> 32) | 1u;
    for (int i = J - 1; i > 0; --i) {
      x = x * 1664525u + 1013904223u;
      const int k = static_cast<int>(__umulhi(x ^ (x >> 15), static_cast<uint32_t>(i + 1)));
      const int a = prio_ld<PB>(sp, i), b = prio_ld<PB>(sp, k);
      prio_st<PB>(sp, i, b);
      prio_st<PB>(sp, k, a);
    }
  }
  __syncthreads();
  const int wo = static_cast<int>(s.stride_o >> 2), wp = static_cast<int>(s.stride_p >> 2);  // strides are multiples of 32 B
  const uint32_t seed_lo = static_cast<uint32_t>(s.seed) ^ static_cast<uint32_t>(s.seed >> 32) * 0x9e3779b1u;
  // write-out, all threads busy: the (row, word) pairs of the CTA are dealt round-robin
  const int rows = static_cast<int>(min(static_cast<long long>(T), s.chains - c0));
  for (int x = threadIdx.x; x < rows * wo; x += T) {
    const int r = x / wo, w = x - r * wo;
    const uint8_t* rp = sm_rows + static_cast<size_t>(r) * row_p;
    const uint64_t gid = s.chain_base + static_cast<uint64_t>(c0 + r);
    uint32_t v = 0;
    if (w * 4 < J) {
      const uint32_t g32 = static_cast<uint32_t>(gid) * 0x9e3779b1u ^ static_cast<uint32_t>(gid >> 32) ^ seed_lo;
      const uint32_t h0 = hash32(g32 + 2u * w), h1 = hash32(g32 + 2u * w + 1u);
      const uint32_t hn = s.nodes > 1 ? hash32(~g32 + w) : 0u;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int i = w * 4 + q;
        if (i < J) {
          const int j = POS ? prio_ld<PB>(rp, i) : i;
          const uint32_t f = ((q & 2) ? h1 : h0) >> (16 * (q & 1)) & 0xffffu;   // 16 random bits per byte
          uint32_t ob = vopt_s[j * kSlots + ((f * nval_s[j]) >> 16)];
          if (s.nodes > 1) ob = (ob & 7u) | ((((hn >> (8 * q)) & 0xffu) * static_cast<uint32_t>(s.nodes) >> 8) << 3);
          v |= ob << (8 * q);
        }
      }
    }
    reinterpret_cast<uint32_t*>(s.cur_o + (c0 + r) * s.stride_o)[w] = v;
  }
  for (int x = threadIdx.x; x < rows * wp; x += T) {
    const int r = x / wp, w = x - r * wp;
    const uint8_t* rp = sm_rows + static_cast<size_t>(r) * row_p;
    reinterpret_cast<uint32_t*>(s.cur_p + (c0 + r) * s.stride_p)[w] =
        (w * 4 < row_p) ? reinterpret_cast<const uint32_t*>(rp)[w] : 0u;
  }
}

__device__ __forceinline__ void copy_row16(uint8_t* dst, const uint8_t* src, int bytes, int lane) {
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
  uint4* d4 = reinterpret_cast<uint4*>(dst);
  for (int i = lane; i * 16 < bytes; i += 32) d4[i] = s4[i];
}

// ---- propose: warp per chain
template <int PB>
__global__ void k_propose(SearchDev s, int round) {
  const int lane = threadIdx.x & 31;
  const long long c = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (c >= s.chains) return;
  const uint8_t* co = s.cur_o + c * s.stride_o;
  const uint8_t* cp = s.cur_p + c * s.stride_p;
  uint8_t* po = s.prop_o + c * s.stride_o;
  uint8_t* pp = s.prop_p + c * s.stride_p;
  copy_row16(po, co, static_cast<int>(s.stride_o), lane);
  copy_row16(pp, cp, static_cast<int>(s.stride_p), lane);
  __syncwarp();
  const uint64_t gid = s.chain_base + static_cast<uint64_t>(c);
  const uint64_t r0 = rng_u64(s.seed, gid, 4ull * round + 0);
  const uint64_t r1 = rng_u64(s.seed, gid, 4ull * round + 1);
  const uint64_t r2 = rng_u64(s.seed, gid, 4ull * round + 2);
  const uint32_t kind = bounded(r0, 100);
  const int J = s.J;
  if (s.nodes > 1 && kind >= 85) {
    // move one job to another node (milp.py:117-137: exactly one node per task)
    if (lane == 0) {
      const int j = bounded(r1, J);
      const uint8_t curv = co[j];
      int nn = bounded(r2, s.nodes - 1);
      if (nn >= (curv >> 3)) ++nn;
      po[j] = static_cast<uint8_t>((curv & 7) | (nn << 3));
    }
    return;
  }
  if (kind < 30) {
    // change one job's option (keeping its node)
    const int j = bounded(r1, J);
    const int n = s.nvalid[j];
    if (n > 1) {
      if (lane == 0) {
        int pick = bounded(r2, n - 1);
        const uint8_t curv = co[j];
        const uint8_t node_bits = s.nodes > 1 ? (curv & 0xf8) : 0;
        const uint8_t cur_opt = s.nodes > 1 ? (curv & 7) : curv;
        uint8_t nv = s.vopt[j * kSlots + pick];
        if (nv == cur_opt) nv = s.vopt[j * kSlots + n - 1];
        po[j] = nv | node_bits;
      }
      return;
    }
  }
  const int a = bounded(r1, J);
  int b = bounded(r2, J - 1);
  if (b >= a) ++b;
  if (J < 2) return;
  if (kind < 65) {
    // swap two priorities
    if (lane == 0) {
      const int va = prio_ld<PB>(cp, a), vb = prio_ld<PB>(cp, b);
      prio_st<PB>(pp, a, vb);
      prio_st<PB>(pp, b, va);
    }
  } else {
    // take the job at position a and re-insert it at position b
    if (a < b) {
      for (int i = a + lane; i < b; i += 32) prio_st<PB>(pp, i, prio_ld<PB>(cp, i + 1));
    } else {
      for (int i = b + 1 + lane; i <= a; i += 32) prio_st<PB>(pp, i, prio_ld<PB>(cp, i - 1));
    }
    if (lane == 0) prio_st<PB>(pp, b, prio_ld<PB>(cp, a));
  }
}

// ---- keep the incumbent encoding when the key improved (one warp)
__global__ void k_keep_best(SearchDev s, const uint8_t* rows_o, const uint8_t* rows_p) {
  const int lane = threadIdx.x & 31;
  const unsigned long long key = s.keys[0];
  if (key >= s.keys[1]) return;
  const uint64_t id = key & 0xffffffffull;
  const uint64_t base = s.chain_base & 0xffffffffull;
  const long long c = static_cast<long long>((id - base) & 0xffffffffull);
  if (c < 0 || c >= s.chains) return;
  copy_row16(s.best_o, rows_o + c * s.stride_o, static_cast<int>(s.stride_o), lane);
  copy_row16(s.best_p, rows_p + c * s.stride_p, static_cast<int>(s.stride_p), lane);
  __syncwarp();
  if (lane == 0) s.keys[1] = key;
}

// ---- Metropolis acceptance: warp per chain
__global__ void k_accept(SearchDev s, int round, float temperature) {
  const int lane = threadIdx.x & 31;
  const long long c = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (c >= s.chains) return;
  const float pm = s.prop_mk[c], cm = s.cur_mk[c];
  bool acc = pm <= cm;
  if (!acc && temperature > 0.f && isfinite(pm)) {
    const uint64_t gid = s.chain_base + static_cast<uint64_t>(c);
    const uint64_t r = rng_u64(s.seed, gid, 4ull * round + 3);
    const float u = (static_cast<uint32_t>(r >> 40) + 0.5f) * (1.0f / 16777216.0f);
    acc = u < __expf(-(pm - cm) / temperature);
  }
  if (!acc) return;
  copy_row16(s.cur_o + c * s.stride_o, s.prop_o + c * s.stride_o, static_cast<int>(s.stride_o), lane);
  copy_row16(s.cur_p + c * s.stride_p, s.prop_p + c * s.stride_p, static_cast<int>(s.stride_p), lane);
  if (lane == 0) s.cur_mk[c] = pm;
}

// ---- overwrite chains [first, first+copies) with one candidate (warp per chain)
__global__ void k_inject(SearchDev s, const uint8_t* cand_o, const uint8_t* cand_p, long long first, int copies) {
  const int lane = threadIdx.x & 31;
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (w >= copies) return;
  const long long c = first + w;
  copy_row16(s.cur_o + c * s.stride_o, cand_o, static_cast<int>(s.stride_o), lane);
  copy_row16(s.cur_p + c * s.stride_p, cand_p, static_cast<int>(s.stride_p), lane);
}

// ---- tournament resampling ("go with the winners"): every chain draws a random rival and, if the
// rival's current makespan is strictly better, continues from a copy of the rival's candidate.
// Two passes through the proposal buffers (then the host swaps the buffer roles), so no chain is
// read while it is being overwritten.  Warp per chain.
template <int PB>
__global__ void k_resample(SearchDev s, int round) {
  const int lane = threadIdx.x & 31;
  const long long c = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (c >= s.chains) return;
  const uint64_t gid = s.chain_base + static_cast<uint64_t>(c);
  const uint64_t r = rng_u64(s.seed ^ 0x7e57a11ull, gid, static_cast<uint64_t>(round));
  const long long d = bounded(r, static_cast<uint32_t>(s.chains));
  const long long src = (s.cur_mk[d] < s.cur_mk[c]) ? d : c;
  copy_row16(s.prop_o + c * s.stride_o, s.cur_o + src * s.stride_o, static_cast<int>(s.stride_o), lane);
  copy_row16(s.prop_p + c * s.stride_p, s.cur_p + src * s.stride_p, static_cast<int>(s.stride_p), lane);
  if (lane == 0) s.prop_mk[c] = s.cur_mk[src];
}

// =====================================================================================================
// Large J: schedule-order ("position-major") populations.
//
// When a candidate's two rows no longer fit in shared memory (J beyond ~450 with u16 priorities) the
// search keeps its population with opt stored BY POSITION — opt[i] is the option of the job scheduled
// i-th, prio[i] that job — so a candidate is simply a sequence of (job, option) pairs.  Both rows are
// then consumed in order: they stream through registers with 256-bit loads, no shared-memory tile is
// needed (16 warps per SM at any J) and a move is a patch of one or two positions of the streams.
// The encoding is internal to the search: candidates enter (warm start, injected seeds) and leave
// (sb_search_best) in the job-indexed encoding of the ABI; sb_api.cu converts on the host.
// =====================================================================================================
template <int PB>
__global__ void k_init_population_pos(SearchDev s) {
  const long long c = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (c >= s.chains) return;
  uint8_t* orow = s.cur_o + c * s.stride_o;
  uint8_t* prow = s.cur_p + c * s.stride_p;
  const uint64_t gid = s.chain_base + static_cast<uint64_t>(c);
  for (int j = 0; j < s.J; ++j) prio_st<PB>(prow, j, j);
  for (int i = s.J - 1; i > 0; --i) {
    const uint64_t r = rng_u64(s.seed, gid, 0x200000000ull + i);
    const int k = bounded(r, i + 1);
    const int a = prio_ld<PB>(prow, i), b = prio_ld<PB>(prow, k);
    prio_st<PB>(prow, i, b);
    prio_st<PB>(prow, k, a);
  }
  for (int i = 0; i < s.J; ++i) {
    const int j = prio_ld<PB>(prow, i);
    const uint64_t r = rng_u64(s.seed, gid, 0x100000000ull + j);
    uint8_t ob = s.vopt[j * kSlots + bounded(r, s.nvalid[j])];
    if (s.nodes > 1) ob = static_cast<uint8_t>((ob & 7) | (bounded(rng_u64(s.seed, gid, 0x300000000ull + j), s.nodes) << 3));
    orow[i] = ob;
  }
}

// k_search_pos with the table split over a CTA pair: entries per half (a multiple of 4 = 16 bytes for TMA)
__host__ __device__ inline uint32_t pos_tab_half(int J, int SG) {
  const uint32_t n = static_cast<uint32_t>(J) * static_cast<uint32_t>(SG);
  return ((n + 1u) / 2u + 3u) & ~3u;
}

struct PosArgs {
  const float* tab;
  int J, SG, nodes;
  uint8_t* opt;   // [chains][stride_o], by position
  uint8_t* prio;  // [chains][stride_p]
  long long chains, first;
  long long stride_o, stride_p;
  unsigned long long* best_key;
  uint32_t id_base;
  int eval_only;  // 1: score the rows as they are and store cur_mk (initialisation, injected rows)
  int one;
  SearchFuse sf;
  const float* w;  // obj_weights(OBJ): job weights [J], zero-padded to a multiple of 4 (16 bytes)
  const float* d;  // obj_due(OBJ): job due dates (or tails) [J], padded the same way
  const float* r;  // R: job release dates [J], padded the same way
  const float* p;  // obj_penalty(OBJ): job late penalties [J], padded the same way
  int K;           // obj_scenario(OBJ): the scenario tables at tab, [K][J][SG] (last: the other fields keep their offsets)
  int pad;         // keeps the struct free of implicit padding: a padding hole changes the code of every kernel taking it
};

struct PosMove {
  int kind;    // 0 none, 1 option byte at position a becomes oa, 2 positions a and b exchange (job, option)
  int a, b;
  int va, vb;  // jobs at a, b
  int oa, ob;  // option bytes at a, b (kind 1: oa = the new byte)
};

template <int PB>
__device__ __forceinline__ PosMove make_pos_move(const SearchFuse& sf, int round, int J, uint64_t gid,
                                                 const uint8_t* og, const uint8_t* pg) {
  PosMove m;
  m.kind = 0; m.a = m.b = m.va = m.vb = m.oa = m.ob = 0;
  const uint64_t r0 = rng_u64(sf.seed, gid, 4ull * round + 0);
  const uint64_t r1 = rng_u64(sf.seed, gid, 4ull * round + 1);
  const uint64_t r2 = rng_u64(sf.seed, gid, 4ull * round + 2);
  const uint32_t kind = bounded(r0, 100);
  if (sf.nodes > 1 && kind >= 85) {  // move the job at a random position to another node
    const int p = bounded(r1, J);
    const int cur = og[p];
    int nn = bounded(r2, sf.nodes - 1);
    if (nn >= (cur >> 3)) ++nn;
    m.kind = 1; m.a = p; m.oa = (cur & 7) | (nn << 3);
    return m;
  }
  if (kind < 30) {  // change the option of the job at a random position (keeping its node)
    const int p = bounded(r1, J);
    const int j = prio_ld<PB>(pg, p);
    const int n = sf.nvalid[j];
    if (n > 1) {
      const int cur = og[p];
      const int node_bits = sf.nodes > 1 ? (cur & 0xf8) : 0;
      const int cur_opt = sf.nodes > 1 ? (cur & 7) : cur;
      int nv = sf.vopt[j * kSlots + bounded(r2, n - 1)];
      if (nv == cur_opt) nv = sf.vopt[j * kSlots + n - 1];
      m.kind = 1; m.a = p; m.oa = nv | node_bits;
      return m;
    }
  }
  if (J < 2) return m;
  const int a = bounded(r1, J);
  int b = bounded(r2, J - 1);
  if (b >= a) ++b;
  m.kind = 2; m.a = a; m.b = b;
  m.va = prio_ld<PB>(pg, a); m.vb = prio_ld<PB>(pg, b);
  m.oa = og[a]; m.ob = og[b];
  return m;
}

// Windowed form (incremental rounds): the first position the move changes lies in [p0, p0 + plen).
template <int PB>
__device__ __forceinline__ PosMove make_pos_move_win(const SearchFuse& sf, int round, int J, uint64_t gid,
                                                     const uint8_t* og, const uint8_t* pg, int p0, int plen) {
  PosMove m;
  m.kind = 0; m.a = m.b = m.va = m.vb = m.oa = m.ob = 0;
  const uint64_t r0 = rng_u64(sf.seed, gid, 4ull * round + 0);
  const uint64_t r1 = rng_u64(sf.seed, gid, 4ull * round + 1);
  const uint64_t r2 = rng_u64(sf.seed, gid, 4ull * round + 2);
  const uint32_t kind = bounded(r0, 100);
  const int a = p0 + static_cast<int>(bounded(r1, plen));
  if (kind < 30) {  // change the option of the job at position a
    const int j = prio_ld<PB>(pg, a);
    const int n = sf.nvalid[j];
    if (n > 1) {
      const int cur = og[a];
      int nv = sf.vopt[j * kSlots + bounded(r2, n - 1)];
      if (nv == cur) nv = sf.vopt[j * kSlots + n - 1];
      m.kind = 1; m.a = a; m.oa = nv;
      return m;
    }
  }
  const int tail = J - p0;
  if (tail < 2) return m;
  int b = p0 + static_cast<int>(bounded(r2, tail - 1));
  if (b >= a) ++b;
  m.kind = 2; m.a = a; m.b = b;
  m.va = prio_ld<PB>(pg, a); m.vb = prio_ld<PB>(pg, b);
  m.oa = og[a]; m.ob = og[b];
  return m;
}

// EVAL: the scoring-only instantiation (sb_eval with SB_FLAG_OPT_BY_POSITION, population scoring after
// initialisation / injection): the move, snapshot and acceptance code folds away at compile time.
// TAB: where the runtime table lives.  0 = this CTA's shared memory.  For tables beyond one SM's shared
// memory (C5 with all 8 strategies: 256 KB) the scoring-only instantiation has two more homes:
// 1 = left in global memory and read through L1 / L2 (the default for such tables: this kernel keeps no tile
// in shared memory, so the launch asks for the whole array as L1);
// 2 = split over the shared memory of a CTA PAIR (cluster of 2): each CTA loads one half with TMA and every
// look-up is a `ld.shared::cluster` to whichever CTA owns the entry (distributed shared memory) — the
// alternative to 1, kept behind a test hook.
// OBJ: the objective (sb_common.cuh), folded by ls_step.  R: no job starts before its release date (SB_FLAG_RELEASE,
// any objective).  The per-job arrays they read (stage_job_array, sb_lane.cuh) follow the table in shared memory with TAB = 0 and are
// read from global memory (ld.global.nc) with TAB = 1 / 2.  obj_scenario(OBJ): the K scenario tables are staged back to
// back (TAB = 0 only), and every evaluation runs one pass of step_obj(OBJ) per table (no snapshots: the host runs
// these forms without incremental rounds) and folds the K scores into the score; the tardiness forms stage and read
// the weights and due dates as the tardiness form does.
template <int PB, bool INT, bool MULTI, bool EVAL = false, int TAB = 0, Obj OBJ = Obj::Makespan, bool R = false>
__global__ void __launch_bounds__(512, 1) k_search_pos(const PosArgs a) {
  static_assert(TAB == 0 || (EVAL && !MULTI), "tables outside the CTA's shared memory: scoring only, one node");
  constexpr bool kScen = obj_scenario(OBJ);
  static_assert(TAB == 0 || !kScen, "the scenario tables live in the CTA's shared memory");
  extern __shared__ __align__(128) uint8_t smem[];
  const int nw = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t tab_all = kScen ? static_cast<uint32_t>(a.J) * a.SG * 4u * static_cast<uint32_t>(a.K)
                                 : static_cast<uint32_t>(a.J) * a.SG * 4u;
  // TAB = 2: rank r of the pair keeps entries [r * half, (r + 1) * half)
  [[maybe_unused]] const uint32_t half = pos_tab_half(a.J, a.SG);
  [[maybe_unused]] const uint32_t rank = TAB == 2 ? cluster_ctarank() : 0u;
  const uint32_t tab_off = TAB == 2 ? rank * half * 4u : 0u;
  const uint32_t tab_bytes = TAB == 1 ? 0u : (TAB == 2 ? (rank == 0 ? half * 4u : tab_all - half * 4u) : tab_all);
  const uint32_t tab_room = TAB == 1 ? 0u : (TAB == 2 ? half * 4u : tab_all);
  constexpr bool kW = obj_weights(OBJ), kD = obj_due(OBJ), kP = obj_penalty(OBJ);
  const uint32_t w_bytes = (kW && TAB == 0) ? ((static_cast<uint32_t>(a.J) * 4u + 15u) & ~15u) : 0u;
  const uint32_t d_bytes = kD ? (kW ? w_bytes : (TAB == 0 ? ((static_cast<uint32_t>(a.J) * 4u + 15u) & ~15u) : 0u)) : 0u;
  const uint32_t r_bytes = (R && TAB == 0) ? ((static_cast<uint32_t>(a.J) * 4u + 15u) & ~15u) : 0u;
  const uint32_t p_bytes = kP ? w_bytes : 0u;  // the penalties come with the weights (obj_weights)
  float* tab_s = reinterpret_cast<float*>(smem);
  [[maybe_unused]] float* w_s = reinterpret_cast<float*>(smem + ((tab_room + 15u) & ~15u));
  [[maybe_unused]] float* d_s = reinterpret_cast<float*>(smem + ((tab_room + 15u) & ~15u) + w_bytes);
  [[maybe_unused]] float* r_s = reinterpret_cast<float*>(smem + ((tab_room + 15u) & ~15u) + w_bytes + d_bytes);
  [[maybe_unused]] float* p_s = reinterpret_cast<float*>(smem + ((tab_room + 15u) & ~15u) + w_bytes + d_bytes + r_bytes);
  uint64_t* bar_tab =
      reinterpret_cast<uint64_t*>(smem + ((tab_room + 15u) & ~15u) + w_bytes + d_bytes + r_bytes + p_bytes);
  const uint32_t node_bytes = MULTI ? static_cast<uint32_t>(a.nodes) * 1024u : 0u;
  float4* node_s = reinterpret_cast<float4*>(reinterpret_cast<uint8_t*>(bar_tab) + 16 + static_cast<size_t>(warp) * node_bytes);
  if (threadIdx.x == 0) {
    mbar_init(bar_tab, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if constexpr (TAB != 1) {
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(bar_tab, tab_bytes + w_bytes + d_bytes + r_bytes + p_bytes);
      const uint8_t* src = reinterpret_cast<const uint8_t*>(a.tab) + tab_off;
      for (uint32_t off = 0; off < tab_bytes; off += 32768u) tma_bulk_g2s(smem + off, src + off, min(32768u, tab_bytes - off), bar_tab);
      if constexpr (kW && TAB == 0) stage_job_array(reinterpret_cast<uint8_t*>(w_s), a.w, w_bytes, bar_tab);
      if constexpr (kD && TAB == 0) stage_job_array(reinterpret_cast<uint8_t*>(d_s), a.d, d_bytes, bar_tab);
      if constexpr (R && TAB == 0) stage_job_array(reinterpret_cast<uint8_t*>(r_s), a.r, r_bytes, bar_tab);
      if constexpr (kP && TAB == 0) stage_job_array(reinterpret_cast<uint8_t*>(p_s), a.p, p_bytes, bar_tab);
    }
  }
  LaneState<INT, MULTI, 0, step_obj(OBJ), TAB == 0 ? 1 : 2, R> st;
  st.tab = tab_s;
  if constexpr (kW) st.wt = TAB == 0 ? w_s : a.w;
  if constexpr (kD) st.dd = TAB == 0 ? d_s : a.d;
  if constexpr (R) st.rr = TAB == 0 ? r_s : a.r;
  if constexpr (kP) st.pp = TAB == 0 ? p_s : a.p;
  st.SG = a.SG;
  st.one = a.one;
  st.orow = nullptr;
  st.ns = node_s + lane;
  if constexpr (TAB != 1) mbar_wait(bar_tab, 0);
  // TAB = 2: both halves are in place once the pair has met; the window addresses of the two halves, the
  // upper one biased so that (entry index * 4) can be added to either
  [[maybe_unused]] uint32_t base_lo = 0, base_hi = 0;
  if constexpr (TAB == 2) {
    cluster_sync_all();
    base_lo = cluster_map_shared(smem_u32(tab_s), 0u);
    base_hi = cluster_map_shared(smem_u32(tab_s), 1u) - half * 4u;
  }
  auto lookup = [&](int j, int o) -> float {
    if constexpr (TAB == 0) {
      return st.lookup_rt(j, o);
    } else if constexpr (TAB == 1) {
      return __ldg(a.tab + static_cast<uint32_t>(j * a.SG + o));
    } else {
      const uint32_t idx = static_cast<uint32_t>(j * a.SG + o);
      const uint32_t addr = (idx >= half ? base_hi : base_lo) + idx * 4u;
      float v;
      asm("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(addr));
      return v;
    }
  };

  const int J = a.J;
  constexpr int PCH = PB;  // prio chunks (256-bit loads) per 32 positions
  const long long ntiles = (a.chains + 31) / 32;
  for (long long tile = static_cast<long long>(blockIdx.x) * nw + warp; tile < ntiles;
       tile += static_cast<long long>(gridDim.x) * nw) {
    const long long c = a.first + tile * 32 + lane;
    const bool active = tile * 32 + lane < a.chains;
    // lanes beyond the end of the population shadow lane 0's chain (read-only): the evaluation below then runs
    // converged on valid rows in every lane
    const long long cr = active ? c : a.first + tile * 32;
    uint8_t* og = a.opt + cr * a.stride_o;
    uint8_t* pg = a.prio + cr * a.stride_p;
    // both rows stream through registers, with the proposed move patched into the chunks.  Incremental
    // rounds: `oc0` > 0 resumes at that 32-position block from the snapshot in front of it (buffer bit of
    // `par`), `save` stores the state in front of every later window boundary into the other buffer
    // (see SearchFuse::snap; a window is `wblk` blocks, chosen so that there are at most 32 windows).
    auto pass = [&](const PosMove& mv, int oc0, uint32_t par, bool save, float* snap_t, int wblk) -> float {
      const int nout = (J + 31) / 32;  // outer iterations of 32 positions
      if (oc0 == 0) {
        st.reset(a.nodes);
      } else {
        const int b = oc0 / wblk - 1;
        const float* sp = snap_t + ((b * 2 + ((par >> b) & 1u)) * 9) * 32 + lane;
#pragma unroll
        for (int i = 0; i < 8; ++i) st.f[i] = __ldcg(sp + i * 32);
        st.mk = __ldcg(sp + 8 * 32);
        st.pend = 0.f;
      }
      PrioChunk qo = ld_prio32<false>(og + oc0 * 32);
      PrioChunk qp[PCH];
#pragma unroll
      for (int h = 0; h < PCH; ++h) qp[h] = ld_prio32<false>(pg + (oc0 * PCH + h) * 32);
      for (int oc = oc0; oc < nout; ++oc) {
        if (save && oc > oc0 && oc % wblk == 0) {
          const int b = oc / wblk - 1;
          float* sp = snap_t + ((b * 2 + (((par >> b) & 1u) ^ 1u)) * 9) * 32 + lane;
#pragma unroll
          for (int i = 0; i < 8; ++i) __stcg(sp + i * 32, st.f[i]);
          __stcg(sp + 8 * 32, st.running());
        }
        PrioChunk no = qo, np[PCH];
#pragma unroll
        for (int h = 0; h < PCH; ++h) np[h] = qp[h];
        if (oc + 1 < nout) {
          no = ld_prio32<false>(og + (oc + 1) * 32);
#pragma unroll
          for (int h = 0; h < PCH; ++h)
            if (((oc + 1) * PCH + h) * (32 / PB) < J) np[h] = ld_prio32<false>(pg + ((oc + 1) * PCH + h) * 32);
        }
        if (mv.kind == 1) {
          patch_chunk<1>(qo, oc, mv.a, mv.oa);
        } else if (mv.kind == 2) {
          patch_chunk<1>(qo, oc, mv.a, mv.ob);
          patch_chunk<1>(qo, oc, mv.b, mv.oa);
#pragma unroll
          for (int h = 0; h < PCH; ++h) {
            patch_chunk<PB>(qp[h], oc * PCH + h, mv.a, mv.vb);
            patch_chunk<PB>(qp[h], oc * PCH + h, mv.b, mv.va);
          }
        }
        const int base = oc * 32;
        if (base + 32 <= J) {
#pragma unroll
          for (int t = 0; t < 32; ++t) {
            const int j = prio_at<PB>(qp[(t * PB) / 32].w, t % (32 / PB));
            const int o = prio_at<1>(qo.w, t);
            st.step_resolved(o, lookup(j, o), t & 1, st.lookup_w(j), st.lookup_d(j), st.lookup_r(j), st.lookup_p(j));
          }
        } else {
#pragma unroll
          for (int t = 0; t < 32; ++t) {
            if (base + t < J) {
              const int j = prio_at<PB>(qp[(t * PB) / 32].w, t % (32 / PB));
              const int o = prio_at<1>(qo.w, t);
              st.step_resolved(o, lookup(j, o), t & 1, st.lookup_w(j), st.lookup_d(j), st.lookup_r(j),
                               st.lookup_p(j));
            }
          }
        }
        qo = no;
#pragma unroll
        for (int h = 0; h < PCH; ++h) qp[h] = np[h];
      }
      return st.result(a.nodes);
    };
    auto evaluate = [&](const PosMove& mv, int oc0, uint32_t par, bool save, float* snap_t, int wblk) -> float {
      if constexpr (kScen) {
        float score = 0.f;
        for (int k = 0; k < a.K; ++k) {
          st.tab = tab_s + static_cast<size_t>(k) * J * a.SG;
          score = scenario_fold<OBJ>(score, pass(mv, 0, par, false, snap_t, wblk));
        }
        return score;
      } else {
        return pass(mv, oc0, par, save, snap_t, wblk);
      }
    };
    PosMove none;
    none.kind = 0; none.a = none.b = none.va = none.vb = none.oa = none.ob = 0;
    // sf.nrounds rounds per launch: an accepted move is written to the rows, which the next round streams
    // again; the lane that lowers the global best key stops moving (see k_eval_tiles).  eval_only: one pass that
    // scores the rows as they are.  The evaluation has ONE call site (the kernel becomes instruction-fetch
    // bound when the unrolled 32-step body is inlined several times): the scoring pass of eval_only, the
    // unmodified pass that fills the snapshots (r = -1), the rounds and the verify hook's recomputation all go
    // through it.
    float cm = (active && !EVAL) ? a.sf.cur_mk[c] : 0.f;
    bool moving = active && !EVAL;  // false from the round in which this lane lowers the global best key
    const uint64_t gid = a.sf.chain_base + static_cast<uint64_t>(c);
    // incremental rounds (one node): windows of wblk 32-position blocks, at most 32 of them
    const int nout_all = (J + 31) / 32;
    const int wblk = (nout_all + 31) / 32;
    const int nwin = (nout_all + wblk - 1) / wblk;
    const bool win = !EVAL && !MULTI && a.sf.win != 0 && nwin >= 2;
    const bool inc = win && a.sf.snap != nullptr;
    float* snap_t = inc ? a.sf.snap + static_cast<size_t>(tile) * (static_cast<size_t>(nwin - 1) * 2 * 9 * 32) : nullptr;
    uint32_t par = 0;
    [[maybe_unused]] const uint32_t inc_bits = EVAL ? 0u : launch_incumbent_bits(a.sf);
    const int r_end = EVAL ? 1 : a.sf.nrounds;
#pragma unroll 1
    for (int r = inc ? -1 : 0; r < r_end; ++r) {
      const int round = a.sf.round + r;
      const bool fill = r < 0;  // unmodified pass: buffer 0 of every boundary
      int w0 = 0;
      if (win && !fill) {
        const uint64_t wr = rng_u64(a.sf.seed ^ 0x31d0ull, a.sf.chain_base + static_cast<uint64_t>(a.first + tile * 32),
                                    static_cast<uint64_t>(round));
        w0 = draw_window(wr, nwin, a.sf.win_bias);
      }
      PosMove mv = none;
      if (moving && !fill) {
        if (win) {
          const int p0 = w0 * wblk * 32;
          mv = make_pos_move_win<PB>(a.sf, round, J, gid, og, pg, p0, min(wblk * 32, J - p0));
        } else {
          mv = make_pos_move<PB>(a.sf, round, J, gid, og, pg);
        }
      }
      float mk = 0.f;
      const int trips = (inc && !fill && a.sf.verify_bad != nullptr) ? 2 : 1;
#pragma unroll 1
      for (int trip = 0; trip < trips; ++trip) {
        const float got = evaluate(mv, (inc && trip == 0) ? w0 * wblk : 0, fill ? ~0u : par, inc && trip == 0, snap_t, wblk);
        if (trip == 0) mk = got;
        else if (active && __float_as_uint(got) != __float_as_uint(mk)) atomicAdd(a.sf.verify_bad, 1ull);
      }
      if (fill) continue;
      if (EVAL) {
        if (active) a.sf.cur_mk[c] = mk;
      } else if (moving) {
        bool acc = mk <= cm;
        const float temp = a.sf.temperature[r];
        if (!acc && temp > 0.f && isfinite(mk)) {
          const uint64_t rr = rng_u64(a.sf.seed, gid, 4ull * round + 3);
          const float u = (static_cast<uint32_t>(rr >> 40) + 0.5f) * (1.0f / 16777216.0f);
          acc = u < __expf(-(mk - cm) / temp);
        }
        if (acc && mv.kind != 0) {
          if (mv.kind == 1) {
            og[mv.a] = static_cast<uint8_t>(mv.oa);
          } else {
            og[mv.a] = static_cast<uint8_t>(mv.ob);
            og[mv.b] = static_cast<uint8_t>(mv.oa);
            prio_st<PB>(pg, mv.a, mv.vb);
            prio_st<PB>(pg, mv.b, mv.va);
          }
          a.sf.cur_mk[c] = mk;
          cm = mk;
          if (inc) par ^= (w0 + 1 < nwin) ? (~0u << w0) : 0u;  // the boundary states this proposal wrote are current now
        } else if (!acc) {
          mk = cm;
        }
      }
      if (a.best_key != nullptr) fold_best(a.best_key, active, mk, a.id_base + static_cast<uint32_t>(tile * 32 + lane), lane);
      if constexpr (!EVAL) {
        if (active && __float_as_uint(mk) < inc_bits) moving = false;  // see launch_incumbent_bits
      }
    }
  }
  if (a.sf.keep.counter != nullptr) keep_best_tail(a.sf);
  // the partner may still be reading this CTA's half of the table
  if constexpr (TAB == 2) cluster_sync_all();
}

// ------------------------------------------------------------------------------------------ host
static int warp_grid(long long warps, int threads) {
  long long blocks = (warps * 32 + threads - 1) / threads;
  return static_cast<int>(blocks < 1 ? 1 : blocks);
}

static int init_row(int bytes) {
  int r16 = (bytes + 15) / 16;
  if ((r16 & 1) == 0) r16 += 1;  // odd multiple of 16 B: the threads' rows start in different banks
  return r16 * 16;
}

// Returns cudaErrorNotSupported when not even 32 rows fit in shared memory (J beyond ~2300): the caller
// then zero-fills the rows and runs the per-thread global-memory kernel.
template <bool POS>
static cudaError_t init_population_smem(const SearchDev& s, cudaStream_t st) {
  const int row_p = init_row(s.J * s.pb);
  const size_t lists = static_cast<size_t>(s.J) * (kSlots + 1);  // staged option lists
  int threads = 128;
  while (threads >= 32 && static_cast<size_t>(threads) * row_p + lists > 48 * 1024) threads >>= 1;
  if (threads < 32) {
    threads = 32;
    if (static_cast<size_t>(threads) * row_p + lists > 220 * 1024) return cudaErrorNotSupported;
  }
  const size_t smem = static_cast<size_t>(threads) * row_p + lists;
  const int grid = static_cast<int>((s.chains + threads - 1) / threads);
  return launch(with_pb(s.pb, [](auto PB) { return k_init_population_smem<PB, POS>; }), grid, threads, smem, st, s,
                row_p);
}

static cudaError_t zero_rows(const SearchDev& s, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(s.cur_o, 0, static_cast<size_t>(s.chains) * s.stride_o, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(s.cur_p, 0, static_cast<size_t>(s.chains) * s.stride_p, st);
  return e;
}

cudaError_t search_init_population(const SearchDev& s, cudaStream_t st) {
  cudaError_t e = init_population_smem<false>(s, st);
  if (e != cudaErrorNotSupported) return e;
  cudaGetLastError();
  if ((e = zero_rows(s, st)) != cudaSuccess) return e;
  const int threads = 128;
  const int grid = static_cast<int>((s.chains + threads - 1) / threads);
  return launch(with_pb(s.pb, [](auto PB) { return k_init_population<PB>; }), grid, threads, 0, st, s);
}

cudaError_t search_propose(const SearchDev& s, int round, cudaStream_t st) {
  const int threads = 256;
  return launch(with_pb(s.pb, [](auto PB) { return k_propose<PB>; }), warp_grid(s.chains, threads), threads, 0, st, s,
                round);
}

cudaError_t search_keep_best(const SearchDev& s, bool from_cur, cudaStream_t st) {
  k_keep_best<<<1, 32, 0, st>>>(s, from_cur ? s.cur_o : s.prop_o, from_cur ? s.cur_p : s.prop_p);
  return cudaGetLastError();
}

cudaError_t search_accept(const SearchDev& s, int round, float temperature, cudaStream_t st) {
  const int threads = 256;
  k_accept<<<warp_grid(s.chains, threads), threads, 0, st>>>(s, round, temperature);
  return cudaGetLastError();
}

cudaError_t search_resample(const SearchDev& s, int round, cudaStream_t st) {
  const int threads = 256;
  return launch(with_pb(s.pb, [](auto PB) { return k_resample<PB>; }), warp_grid(s.chains, threads), threads, 0, st, s,
                round);
}

cudaError_t search_inject(const SearchDev& s, const uint8_t* cand_o, const uint8_t* cand_p, long long first,
                          int copies, cudaStream_t st) {
  const int threads = 256;
  k_inject<<<warp_grid(copies, threads), threads, 0, st>>>(s, cand_o, cand_p, first, copies);
  return cudaGetLastError();
}

cudaError_t search_init_population_pos(const SearchDev& s, cudaStream_t st) {
  cudaError_t e = init_population_smem<true>(s, st);
  if (e != cudaErrorNotSupported) return e;
  cudaGetLastError();
  if ((e = zero_rows(s, st)) != cudaSuccess) return e;
  const int threads = 128;
  const int grid = static_cast<int>((s.chains + threads - 1) / threads);
  return launch(with_pb(s.pb, [](auto PB) { return k_init_population_pos<PB>; }), grid, threads, 0, st, s);
}

// smem: table (+ weights, + due dates, + release dates, + late penalties) + mbarrier + per-warp node states (MULTI)
size_t search_pos_smem(int J, int SG, int nodes, int warps, int arrays) {
  const size_t tab_bytes = (static_cast<size_t>(J) * SG * 4 + 15) & ~size_t(15);
  return tab_bytes + arrays * job_array_bytes(J) + 16 + static_cast<size_t>(warps) * (nodes > 1 ? nodes * 1024u : 0u);
}

size_t scenario_smem(int J, int SG, int K, int nodes, unsigned flags, Obj obj) {
  return search_pos_smem(J, SG * K, nodes, 16, job_arrays(obj, flags));
}

using PosKernel = void (*)(PosArgs);

// Scoring-only launches with the table outside the CTA's own shared memory (TAB = tab_home = 1 / 2 of k_search_pos).
static cudaError_t eval_pos_far_launch(const Device& dev, const PosArgs& a, int tab_home, int pb, unsigned flags,
                                       Obj obj, cudaStream_t st) {
  const int warps = 16;
  const size_t smem = tab_home == 2 ? static_cast<size_t>(pos_tab_half(a.J, a.SG)) * 4 + 16 : 16;
  if (smem > dev.smem_optin) return cudaErrorNotSupported;
  const long long ntiles = (a.chains + 31) / 32;
  const long long ctas = (ntiles + warps - 1) / warps;
  const PosKernel kern = with_eval_types(pb, flags, obj, [&](auto PB, auto INT, auto OBJ, auto R) {
    return tab_home == 2 ? k_search_pos<PB, INT, false, true, 2, OBJ, R>
                         : k_search_pos<PB, INT, false, true, 1, OBJ, R>;
  });
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(warps * 32);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr;
  if (tab_home == 2) {
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = 2; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    cfg.gridDim = dim3(2);
    int pairs = 0;
    e = cudaOccupancyMaxActiveClusters(&pairs, kern, &cfg);
    if (e != cudaSuccess) return e;
    if (pairs < 1) return cudaErrorNotSupported;
    const long long want = (ctas + 1) / 2;
    cfg.gridDim = dim3(static_cast<unsigned>(2 * (want < pairs ? want : pairs)));
  } else {
    // nothing but an mbarrier in shared memory: leave the SM's array to L1, which caches the table
    e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 0);
    if (e != cudaSuccess) return e;
    cfg.gridDim = dim3(static_cast<unsigned>(ctas < dev.sm_count ? ctas : dev.sm_count));
  }
  return cudaLaunchKernelEx(&cfg, kern, a);
}

// tab_home: 0 = the table in every CTA's shared memory (cudaErrorNotSupported when it does not fit);
// scoring only, one node: 2 = split over CTA pairs, 1 = global memory
cudaError_t search_pos_launch(const Device& dev, const SearchDev& s, const float* tab, const float* w, const float* d,
                              const float* r, const float* p, int SG, unsigned flags, Obj obj, long long first,
                              long long count, bool eval_only, const SearchFuse& sf, cudaStream_t st, int tab_home,
                              int K) {
  if (count <= 0) return cudaSuccess;
  PosArgs a;
  a.tab = tab; a.J = s.J; a.SG = SG; a.nodes = s.nodes;
  a.opt = s.cur_o; a.prio = s.cur_p;
  a.chains = count; a.first = first;
  a.stride_o = s.stride_o; a.stride_p = s.stride_p;
  a.best_key = s.keys;
  a.id_base = static_cast<uint32_t>(s.chain_base + static_cast<uint64_t>(first));
  a.eval_only = eval_only ? 1 : 0;
  a.one = 1;
  a.sf = sf;
  a.w = w;
  a.d = d;
  a.r = r;
  a.p = p;
  a.K = K;
  a.pad = 0;
  const bool multi = s.nodes > 1;
  const bool scen = obj_scenario(obj);
  if (tab_home != 0) {
    if (!eval_only || multi || scen) return cudaErrorNotSupported;
    return eval_pos_far_launch(dev, a, tab_home, s.pb, flags, obj, st);
  }
  const int warps = 16;
  const size_t smem = scen ? scenario_smem(s.J, SG, K, s.nodes, flags, obj)
                           : search_pos_smem(s.J, SG, s.nodes, warps, job_arrays(obj, flags));
  if (smem > dev.smem_optin) return cudaErrorNotSupported;
  const long long ntiles = (count + 31) / 32;
  const long long ctas = (ntiles + warps - 1) / warps;
  const int grid = static_cast<int>(ctas < dev.sm_count ? ctas : dev.sm_count);
  const auto pick = [&](auto PB, auto INT, auto OBJ, auto R) -> PosKernel {
    return with_bool(multi, [&](auto MULTI) {
      return with_bool(eval_only, [&](auto EVAL) -> PosKernel {
        return k_search_pos<PB, INT, MULTI, EVAL, 0, OBJ, R>;
      });
    });
  };
  const PosKernel kern = scen ? with_scenario_types(s.pb, flags, obj, pick) : with_eval_types(s.pb, flags, obj, pick);
  return launch(kern, grid, warps * 32, smem, st, a);
}

// Where the position-major scoring kernel keeps a table of J x SG entries: 0 = every CTA's shared memory;
// a one-node table that does not fit there: 1 = global memory, read through L1 / L2 (with no tile in shared
// memory the SM's whole array is L1); -1 = nowhere (multi-node table beyond shared memory).
// HOOK_TABLE_PAIR forces 2 (split over CTA pairs: scattered 4-byte ld.shared::cluster), HOOK_TABLE_GLOBAL forces 1.
int eval_pos_home(const Device& dev, int J, int SG, int nodes, unsigned flags, Obj obj, int K) {
  // the scenario tables: shared memory or nowhere (check_per_job has already held them to scenario_smem)
  if (obj_scenario(obj))
    return !(flags & (HOOK_TABLE_PAIR | HOOK_TABLE_GLOBAL)) && scenario_smem(J, SG, K, nodes, flags, obj) <= dev.smem_optin ? 0 : -1;
  const bool pair_ok = nodes == 1 && static_cast<size_t>(pos_tab_half(J, SG)) * 4 + 16 <= dev.smem_optin;
  if (flags & HOOK_TABLE_PAIR) return pair_ok ? 2 : -1;
  if (flags & HOOK_TABLE_GLOBAL) return nodes == 1 ? 1 : -1;
  if (search_pos_smem(J, SG, nodes, 16, job_arrays(obj, flags)) <= dev.smem_optin) return 0;
  return nodes == 1 ? 1 : -1;
}

// sb_eval with SB_FLAG_OPT_BY_POSITION: score caller rows whose opt bytes are in schedule order.
// *path: 5 = table in shared memory, 7 = table split over CTA pairs, 8 = table in global memory.
cudaError_t eval_pos_launch(const Device& dev, const EvalCall& c, cudaStream_t st, int* path) {
  if (c.stride_o % 32 != 0 || reinterpret_cast<uintptr_t>(c.opt) % 32 != 0 || reinterpret_cast<uintptr_t>(c.prio) % 32 != 0)
    return cudaErrorNotSupported;
  const int home = eval_pos_home(dev, c.J, c.SG, c.nodes, c.flags, c.obj, c.K);
  if (home < 0) return cudaErrorNotSupported;
  if (path) *path = home == 0 ? 5 : (home == 2 ? 7 : 8);
  if (c.B <= 0) return cudaSuccess;
  SearchDev s;
  s.J = c.J; s.pb = c.J <= 256 ? 1 : 2; s.nodes = c.nodes;
  s.cur_o = const_cast<uint8_t*>(c.opt);  // eval_only: rows are read, never written
  s.cur_p = const_cast<uint8_t*>(c.prio);
  s.chains = c.B; s.chain_base = c.id_base;
  s.stride_o = c.stride_o; s.stride_p = c.stride_p;
  s.keys = c.best_key;
  SearchFuse sf = {};
  sf.cur_mk = c.out;
  return search_pos_launch(dev, s, c.tab, c.w, c.d, c.r, c.p, c.SG, c.flags, c.obj, 0, c.B, true, sf, st, home, c.K);
}

// Job-indexed opt rows -> schedule order (out[i] = opt[prio[i]]), one warp per candidate: the row is staged in
// shared memory, each lane gathers 4 positions per store.  sb_eval uses it to send job-indexed candidates at
// large J to the position-major kernel.
template <int PB>
__global__ void __launch_bounds__(256) k_opt_by_position(const uint8_t* __restrict__ opt, const uint8_t* __restrict__ prio,
                                                         uint8_t* __restrict__ out, long long B, int J, long long stride_o,
                                                         long long stride_p, int row_s) {
  extern __shared__ __align__(16) uint8_t rows[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  uint8_t* row = rows + static_cast<size_t>(warp) * row_s;
  for (long long b = static_cast<long long>(blockIdx.x) * nw + warp; b < B; b += static_cast<long long>(gridDim.x) * nw) {
    const uint8_t* og = opt + b * stride_o;
    const uint8_t* pg = prio + b * stride_p;
    __syncwarp();
    if ((reinterpret_cast<uintptr_t>(og) & 15u) == 0) {
      for (int i = lane * 16; i < J; i += 32 * 16) *reinterpret_cast<uint4*>(row + i) = __ldg(reinterpret_cast<const uint4*>(og + i));
    } else {
      for (int i = lane; i < J; i += 32) row[i] = og[i];
    }
    __syncwarp();
    uint8_t* dst = out + b * stride_o;
    for (int i = lane * 4; i < J; i += 32 * 4) {
      uint32_t w = 0;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        if (i + t < J) {
          const int j = PB == 1 ? pg[i + t] : reinterpret_cast<const uint16_t*>(pg)[i + t];
          w |= static_cast<uint32_t>(row[j]) << (8 * t);
        }
      }
      *reinterpret_cast<uint32_t*>(dst + i) = w;
    }
  }
}

// rows of `out` have the stride of the opt rows (a multiple of 4 bytes)
cudaError_t opt_by_position_launch(const Device& dev, const EvalCall& c, uint8_t* out, cudaStream_t st) {
  if (c.B <= 0) return cudaSuccess;
  if (c.stride_o % 16 != 0) return cudaErrorNotSupported;
  const int row_s = (c.J + 15) & ~15;
  const int threads = 256;
  const size_t smem = static_cast<size_t>(threads / 32) * row_s;
  if (smem > 48 * 1024) return cudaErrorNotSupported;
  const long long need = (c.B + threads / 32 - 1) / (threads / 32);
  const long long cap = static_cast<long long>(dev.sm_count) * 8;
  const int grid = static_cast<int>(need < cap ? need : cap);
  return launch(with_pb(c.J <= 256 ? 1 : 2, [](auto PB) { return k_opt_by_position<PB>; }), grid, threads, smem, st,
                c.opt, c.prio, out, c.B, c.J, c.stride_o, c.stride_p, row_s);
}

}  // namespace sb
