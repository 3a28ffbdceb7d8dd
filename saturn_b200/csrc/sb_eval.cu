// sb_eval.cu — makespan evaluation of list-schedule candidates (the measured hot kernel).
//
// Replaces the arithmetic the reference hands to Gurobi/CBC (saturn/solver/milp.py:321-327):
// instead of branch-and-bound over the MILP of milp.py:96-319, B candidates
// (option vector, priority permutation) are scored in parallel; each score is the makespan the
// MILP's constraints would force for that choice of strategies / GPU counts / nodes / ordering.
//
// Kernel shape (k_eval_tiles):
//   * persistent grid, one CTA per SM, NW warps per CTA; the J x S x 8 runtime table is staged
//     once per CTA into shared memory with TMA bulk copies (cp.async.bulk + mbarrier);
//   * each warp owns a tile of 32 candidates: every lane fetches ITS candidate's opt row with one
//     TMA bulk copy into a padded shared-memory row, or (streamed kernel, rows back to back) lane 0
//     fetches the whole tile with one copy (the opt bytes are gathered by job id, so they must be
//     resident), completion on a per-warp mbarrier — no CTA-wide barrier after
//     start-up.  The prio row is consumed in order, so in the STREAM variant (rows 32-byte
//     aligned) each lane streams it straight from HBM, one full 32-byte sector per lane (two
//     128-bit loads, prefetched 32 steps ahead), and it never touches shared memory: 8.7 KB of smem
//     per warp instead of 17.4 KB -> 16 resident warps per SM instead of 8 (with 2 warps per
//     scheduler, dependency waits leave issue slots empty).  Unaligned rows fall back to
//     the non-STREAM variant (prio rows staged in shared memory, TMA or plain loads);
//   * one candidate per LANE: the 8 slot ready-times live sorted in 8 registers and one
//     scheduling step is a few dozen instructions (sb_common.cuh: ls_step) — fp32 min/max/add and byte
//     indexing only, no tensor cores;
//   * MULTI variant (several nodes, milp.py:117-137: a gang stays inside one node): the sorted
//     state of every node lives in a lane-private shared-memory column (2 x float4 per node,
//     conflict-free); a step loads the state of the job's node, updates it, stores it back;
//   * makespans are written coalesced (128 B per warp); an optional 64-bit arg-min key is
//     folded with one redux + one atomicMin per warp;
//   * OBJ: every kernel here comes in a form per objective (sb_common.cuh: Obj), folded by ls_step; the schedule,
//     and every start, is the same under all of them.  The per-job arrays an objective reads (weights,
//     due dates or tails, late penalties) sit beside the table wherever the table is in shared memory (same TMA
//     phase), and are read from global memory where the table is;
//   * R (SB_FLAG_RELEASE, with any objective): no job starts before its release date.  Every objective form has
//     a release twin; the release dates follow the other per-job arrays, in the same memory and TMA phase.
#include "sb_lane.cuh"

namespace sb {

struct TileArgs {
  const float* tab;  // [J][SG] fp32, SG = S*8
  int J, SG;
  const uint8_t* opt;
  const uint8_t* prio;
  long long B;
  long long stride_o, stride_p;  // bytes between candidate rows in global memory
  int row_o, row_p;              // shared-memory row strides (bytes, odd multiple of 16)
  int copy_o, copy_p;            // bytes per row copy (multiple of 16)
  int use_bulk;                  // rows are 16-byte aligned -> TMA bulk copies
  int nodes;                     // MULTI: number of nodes (2..kMaxNodes)
  float* out;
  unsigned long long* best_key;
  uint32_t id_base;
  long long ntiles;
  int one;  // run-time 1 (see pmov_fma)
  SearchFuse sf;  // SEARCH variant only
  XchgPost xp;    // xp.counter != nullptr: the last CTA to finish posts *best_key to every peer's mailbox
  const float* w;  // obj_weights(OBJ): job weights [J], zero-padded to a multiple of 4 (16 bytes)
  const float* d;  // obj_due(OBJ): job due dates (or tails) [J], padded the same way
  const float* r;  // R: job release dates [J], padded the same way
  // the streamed tile kernel (STREAM, one node, table in shared memory) only; see "Tile boundaries" below
  int packed;    // consecutive candidates' rows lie back to back (stride_o == copy_o == row_o, stride_p == copy_p)
  int stagger;   // start the warps of a CTA at staggered phases
  unsigned long long* tile_wait;  // TILE_DEBUG_TIMING: [0] += fetch-to-wait ns, [1] += tile-loop ns, per warp
  const float* p;  // obj_penalty(OBJ): job late penalties [J], padded like w (last: the other fields keep their offsets)
};

// TABG: the runtime table stays in global memory (read through L1/L2) — for tables larger than the
// shared memory left beside the opt tiles (e.g. J = 1024 with 8 strategies: 256 KB).
template <int PB, bool INT, bool STREAM, bool MULTI, bool SEARCH = false, bool TABG = false, int ADDR = 0,
          Obj OBJ = Obj::Makespan, bool R = false>
__global__ void __launch_bounds__(STREAM ? 512 : 384, 1) k_eval_tiles(const TileArgs a) {
  static_assert(!(SEARCH && (STREAM || TABG)), "the fused search round runs on shared-memory tiles only");
  static_assert(ADDR == 0 || (!TABG && !MULTI && !SEARCH), "ADDR = 1 needs the table and the opt rows in shared memory");
  extern __shared__ __align__(128) uint8_t smem[];
  const int nw = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t tab_bytes = TABG ? 0u : static_cast<uint32_t>(a.J) * a.SG * 4u;  // a multiple of 32 (SG = S * 8)
  // the per-job arrays the objective reads follow the table in the same TMA phase, each padded to 16 bytes: the
  // weights, the due dates (or tails), the release dates, the late penalties (TABG: they all stay in global memory)
  constexpr bool kW = obj_weights(OBJ), kD = obj_due(OBJ), kP = obj_penalty(OBJ);
  const uint32_t w_bytes = (kW && !TABG) ? ((static_cast<uint32_t>(a.J) * 4u + 15u) & ~15u) : 0u;
  const uint32_t d_bytes = kD ? (kW ? w_bytes : (TABG ? 0u : ((static_cast<uint32_t>(a.J) * 4u + 15u) & ~15u))) : 0u;
  const uint32_t r_bytes = (R && !TABG) ? ((static_cast<uint32_t>(a.J) * 4u + 15u) & ~15u) : 0u;
  const uint32_t p_bytes = kP ? w_bytes : 0u;  // the penalties come with the weights (obj_weights)
  float* tab_s = reinterpret_cast<float*>(smem);
  [[maybe_unused]] float* w_s = reinterpret_cast<float*>(smem + tab_bytes);
  [[maybe_unused]] float* d_s = reinterpret_cast<float*>(smem + tab_bytes + w_bytes);
  [[maybe_unused]] float* r_s = reinterpret_cast<float*>(smem + tab_bytes + w_bytes + d_bytes);
  [[maybe_unused]] float* p_s = reinterpret_cast<float*>(smem + tab_bytes + w_bytes + d_bytes + r_bytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ((tab_bytes + w_bytes + d_bytes + r_bytes + p_bytes + 15u) & ~15u));
  uint8_t* tiles = reinterpret_cast<uint8_t*>(bars) + (((1 + nw) * 8 + 15) & ~15);
  const uint32_t node_bytes = MULTI ? static_cast<uint32_t>(a.nodes) * 1024u : 0u;
  const uint32_t tile_bytes = 32u * (a.row_o + (STREAM ? 0 : a.row_p)) + node_bytes;
  uint8_t* wbase = tiles + static_cast<size_t>(warp) * tile_bytes;
  float4* node_s = reinterpret_cast<float4*>(wbase);  // [2*nodes][32] float4, first (16-byte aligned)
  uint8_t* tile_o = wbase + node_bytes;
  uint8_t* tile_p = tile_o + 32u * a.row_o;
  uint64_t* bar_tab = bars;
  uint64_t* bar_w = bars + 1 + warp;

  if (threadIdx.x == 0) {
    mbar_init(bar_tab, 1);
    for (int w = 0; w < nw; ++w) mbar_init(bars + 1 + w, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if constexpr (!TABG) {
    if (threadIdx.x == 0) {
      // stage the runtime table: TMA bulk copies of <= 32 KB each, one mbarrier phase
      mbar_arrive_expect_tx(bar_tab, tab_bytes + w_bytes + d_bytes + r_bytes + p_bytes);
      const uint8_t* src = reinterpret_cast<const uint8_t*>(a.tab);
      for (uint32_t off = 0; off < tab_bytes; off += 32768u) {
        uint32_t n = min(32768u, tab_bytes - off);
        tma_bulk_g2s(smem + off, src + off, n, bar_tab);
      }
      if constexpr (kW) stage_job_array(smem + tab_bytes, a.w, w_bytes, bar_tab);
      if constexpr (kD) stage_job_array(smem + tab_bytes + w_bytes, a.d, d_bytes, bar_tab);
      if constexpr (R) stage_job_array(smem + tab_bytes + w_bytes + d_bytes, a.r, r_bytes, bar_tab);
      if constexpr (kP) stage_job_array(smem + tab_bytes + w_bytes + d_bytes + r_bytes, a.p, p_bytes, bar_tab);
    }
  }

  LaneState<INT, MULTI, ADDR, OBJ, TABG ? 2 : 1, R> st;
  if (TABG) st.tab = a.tab;
  else st.tab = tab_s;
  if constexpr (kW) {
    st.wt = TABG ? a.w : w_s;
    st.wt_s = smem_u32(w_s);
  }
  if constexpr (kD) {
    st.dd = TABG ? a.d : d_s;
    st.dd_s = smem_u32(d_s);
  }
  if constexpr (R) {
    st.rr = TABG ? a.r : r_s;
    st.rr_s = smem_u32(r_s);
  }
  if constexpr (kP) {
    st.pp = TABG ? a.p : p_s;
    st.pp_s = smem_u32(p_s);
  }
  st.SG = a.SG;
  st.one = a.one;
  st.orow = tile_o + lane * a.row_o;
  st.ns = node_s + lane;
  st.orow_s = smem_u32(tile_o + lane * a.row_o);
  st.tab_s = smem_u32(tab_s);
  st.four = static_cast<uint32_t>(a.one) * 4u;

  // Pipelined exchange: warp 0 of CTA 0 folds the keys every rank published for the PREVIOUS round into
  // best_key (lane r loads rank r's mailbox over NVLink, acquire at system scope).  It never blocks in front
  // of its tiles: it looks once here and then once per tile boundary until every rank's round has shown up
  // (a late peer costs this warp one NVLink round trip per look instead of stalling the CTA's slowest
  // warp), and only spins — bounded — after its last tile.  The publish of this round is in the tail.
  bool fold_pending = a.xp.counter != nullptr && a.xp.fold_prev && a.xp.seq > 1 && blockIdx.x == 0 && warp == 0;
  // a look = two loads per lane (round number with acquire, then the key), ISSUED at one tile boundary and
  // CONSUMED at the next: the NVLink round trip overlaps the tile's evaluation instead of stalling this
  // warp — every warp has the same number of tiles, so the folding warp's stalls would be the kernel's tail
  unsigned long long pf_seen = 0ull, pf_key = ~0ull;
  auto look_issue = [&]() {
    if (lane < a.xp.x.world) {
      const unsigned long long* slot = a.xp.x.peer[lane] + ((a.xp.seq - 1) & 1ull) * 2;
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(pf_seen) : "l"(slot + 1) : "memory");
      asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(pf_key) : "l"(slot) : "memory");  // valid iff pf_seen shows the round
    }
  };
  auto fold_keys = [&](unsigned long long k) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, k, d);
      k = o < k ? o : k;
    }
    if (lane == 0) atomicMin(a.best_key, k);
    fold_pending = false;
  };
  auto look_consume = [&]() {  // non-blocking: uses the loads issued one tile ago
    const unsigned long long want = a.xp.seq - 1;
    const bool ok = lane >= a.xp.x.world || pf_seen >= want;
    if (__all_sync(0xffffffffu, ok)) fold_keys(lane < a.xp.x.world ? pf_key : ~0ull);
  };
  auto try_fold = [&](bool block) {
    const unsigned long long want = a.xp.seq - 1;
    unsigned long long k = ~0ull;
    bool ok = true;
    if (lane < a.xp.x.world) {
      const unsigned long long* slot = a.xp.x.peer[lane] + (want & 1ull) * 2;
      unsigned long long seen;
      unsigned spins = 0;
      for (;;) {
        asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(slot + 1) : "memory");
        if (seen >= want || !block || ++spins >= (1u << 22)) break;
        __nanosleep(64);
      }
      ok = seen >= want;
      if (ok) asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(k) : "l"(slot) : "memory");
    }
    ok = __all_sync(0xffffffffu, ok);
    if (!ok) {
      if (block && lane == 0) *a.xp.error = 1;  // a peer never published: report, do not hang
      return;
    }
    fold_keys(k);
  };
  if (fold_pending) look_issue();

  // Tile boundaries of the streamed kernel (kFetch).  Every warp has the same work per tile, so warps that start
  // together reach every tile boundary together, and a whole GPU's row fetches then land on HBM at once while no
  // warp can issue.  Two things shorten and spread that wait:
  //   * packed rows: lane 0 fetches the tile's 32 opt rows with ONE bulk copy into an unpadded tile (row stride
  //     copy_o; the opt bytes are gathered by job id, on random banks at either stride);
  //   * staggered phases: when every warp of the CTA has >= 2 tiles (uniform per CTA), warp w waits before its
  //     first tile, on named barrier p = w % nph, until warp 0 has scored p chunks of its first tile (warp 0 arrives
  //     after chunk p).  Offsets stay under half a tile; the warps then keep them, since they run the same work.
  //     Warp 0 — in CTA 0 the one that folds the peers' keys — is never gated.
  constexpr bool kFetch = STREAM && !MULTI && !TABG && !SEARCH;
  const long long tstride = static_cast<long long>(gridDim.x) * nw;
  const int nfull_ch = a.J / (32 / PB);  // full chunks (32 / PB schedule positions each) of a candidate
  int nph = 1;
  if (kFetch && a.stagger && static_cast<long long>(blockIdx.x) * nw + tstride + nw - 1 < a.ntiles)
    nph = min(min(4, nw), (nfull_ch + 1) / 2);
  // threads of barrier p: warp 0 and the warps w = p, p + nph, ... below nw
  auto gate_count = [&](int p) { return 32u * (1u + static_cast<uint32_t>((nw - 1 - p) / nph + 1)); };
  int arrive_at = nfull_ch + 1;  // the chunk after which warp 0 next arrives (never, unless it gates)
  if (nph > 1) {
    if (warp == 0) {
      arrive_at = 1;
    } else if (warp % nph != 0) {
      named_sync(warp % nph, gate_count(warp % nph));
    }
  }
  unsigned long long t_wait = 0ull, t_loop = 0ull;
  if (kFetch && a.tile_wait != nullptr) t_loop = globaltimer_ns();

  uint32_t phase = 0;
  bool tab_ready = TABG;
  for (long long tile = static_cast<long long>(blockIdx.x) * nw + warp; tile < a.ntiles; tile += tstride) {
    const long long b0 = tile * 32;
    if (!SEARCH && fold_pending) {
      look_consume();
      if (fold_pending) look_issue();
    }
    // the candidate of this lane: consecutive ids, or (search rounds, sf.deal = 1) one id from each of 32
    // far-apart blocks so that successive launches put different chains into one warp
    const long long cand = (SEARCH && a.sf.deal) ? lane * a.ntiles + tile : b0 + lane;
    const bool active = cand < a.B;
    const int nb = SEARCH ? __popc(__ballot_sync(0xffffffffu, active)) : static_cast<int>(min(32ll, a.B - b0));
    const uint8_t* pg = a.prio + cand * a.stride_p;
    // ---- fetch this warp's 32 candidate rows
    __syncwarp();
    PrioChunk q;
    if (a.use_bulk) {
      unsigned long long t_fetch = 0ull;
      if (kFetch && a.tile_wait != nullptr) t_fetch = globaltimer_ns();
      fence_proxy_async();  // order the previous tile's generic-proxy reads before async writes
      if (lane == 0)
        mbar_arrive_expect_tx(bar_w, static_cast<uint32_t>(nb) * (a.copy_o + (STREAM ? 0 : a.copy_p)));
      __syncwarp();
      if (kFetch && a.packed) {
        if (lane == 0) tma_bulk_g2s(tile_o, a.opt + b0 * a.stride_o, static_cast<uint32_t>(nb) * a.copy_o, bar_w);
      } else if (active) {
        tma_bulk_g2s(tile_o + lane * a.row_o, a.opt + cand * a.stride_o, a.copy_o, bar_w);
        if (!STREAM) tma_bulk_g2s(tile_p + lane * a.row_p, pg, a.copy_p, bar_w);
      }
      if (STREAM && active) q = ld_prio32<true>(pg);  // overlaps the TMA wait
      mbar_wait(bar_w, phase);
      phase ^= 1;
      if (kFetch && a.tile_wait != nullptr) t_wait += globaltimer_ns() - t_fetch;
    } else {
      for (int r = 0; r < nb; ++r) {
        const uint8_t* so = a.opt + (b0 + r) * a.stride_o;
        const uint8_t* sp = a.prio + (b0 + r) * a.stride_p;
        for (int x = lane; x < a.J; x += 32) tile_o[r * a.row_o + x] = so[x];
        for (int x = lane; x < a.J * PB; x += 32) tile_p[r * a.row_p + x] = sp[x];
      }
      __syncwarp();
    }
    if (!tab_ready) {
      mbar_wait(bar_tab, 0);
      tab_ready = true;
    }
    // ---- one candidate per lane
    auto evaluate = [&](const uint8_t* prio_row_s) -> float {
      st.reset(a.nodes);
      const int J = a.J;
      if constexpr (STREAM && ADDR == 1) {
        // The look-ups of a step do not depend on the slot state, but each is two dependent shared-memory
        // gathers on random banks.  So the full chunks run in batches of kBatch positions: the gathers of
        // batch n + 1 (all opt bytes, then all runtimes) are issued before the steps of batch n, which read
        // their look-ups from registers.  The last batch of a chunk resolves the first batch of the next
        // full chunk, so the pipeline runs across chunks; a partial last chunk takes the plain steps.
        constexpr int STEPS = 32;
        constexpr int kBatch = 8;  // 90 registers, no spills: within the 128 that 16 warps per SM allow
        const int nch = (J + STEPS - 1) / STEPS, nfull = J / STEPS;
        uint32_t ob[kBatch];
        float rb[kBatch];
        [[maybe_unused]] float wb[kBatch];  // kW: the batch's weights, gathered with its runtimes
        [[maybe_unused]] float db[kBatch];  // kD: the batch's due dates (or tails), likewise
        [[maybe_unused]] float xb[kBatch];  // R: the batch's release dates, likewise
        [[maybe_unused]] float pb[kBatch];  // kP: the batch's late penalties, likewise
        auto resolve = [&](const uint32_t* w) {  // w: the kBatch / 4 words that hold the batch's job ids
          int js[kBatch];
#pragma unroll
          for (int i = 0; i < kBatch; ++i) js[i] = prio_at<1>(w, i);
#pragma unroll
          for (int i = 0; i < kBatch; ++i) ob[i] = st.gather_opt(js[i]);
#pragma unroll
          for (int i = 0; i < kBatch; ++i) rb[i] = st.gather_rt(js[i], ob[i]);
          if constexpr (kW) {
#pragma unroll
            for (int i = 0; i < kBatch; ++i) wb[i] = st.gather_w(js[i]);
          }
          if constexpr (kD) {
#pragma unroll
            for (int i = 0; i < kBatch; ++i) db[i] = st.gather_d(js[i]);
          }
          if constexpr (R) {
#pragma unroll
            for (int i = 0; i < kBatch; ++i) xb[i] = st.gather_r(js[i]);
          }
          if constexpr (kP) {
#pragma unroll
            for (int i = 0; i < kBatch; ++i) pb[i] = st.gather_p(js[i]);
          }
        };
        if (nfull > 0) resolve(q.w);
        // one copy of the chunk loop: it stops early only where warp 0 opens a stagger barrier (first tile)
        int c = 0, stop = min(arrive_at, nfull);
        for (;;) {
        for (; c < stop; ++c) {
          PrioChunk nxt = q;
          if (c + 1 < nch) nxt = ld_prio32<true>(pg + (c + 1) * 32);
          // a partial next chunk is not resolved ahead (its bytes past J are not job ids): the last batch then
          // re-resolves this chunk's first batch, and the result is not used
          const bool ahead = c + 1 < nfull;
          uint32_t head[kBatch / 4];
#pragma unroll
          for (int i = 0; i < kBatch / 4; ++i) head[i] = ahead ? nxt.w[i] : q.w[i];
#pragma unroll
          for (int b = 0; b < STEPS / kBatch; ++b) {
            uint32_t oc[kBatch];
            float rc[kBatch];
            [[maybe_unused]] float wc[kBatch];
            [[maybe_unused]] float dc[kBatch];
            [[maybe_unused]] float xc[kBatch];
            [[maybe_unused]] float pc[kBatch];
#pragma unroll
            for (int i = 0; i < kBatch; ++i) { oc[i] = ob[i]; rc[i] = rb[i]; }
            if constexpr (kW) {
#pragma unroll
              for (int i = 0; i < kBatch; ++i) wc[i] = wb[i];
            }
            if constexpr (kD) {
#pragma unroll
              for (int i = 0; i < kBatch; ++i) dc[i] = db[i];
            }
            if constexpr (R) {
#pragma unroll
              for (int i = 0; i < kBatch; ++i) xc[i] = xb[i];
            }
            if constexpr (kP) {
#pragma unroll
              for (int i = 0; i < kBatch; ++i) pc[i] = pb[i];
            }
            resolve(b + 1 < STEPS / kBatch ? q.w + (b + 1) * (kBatch / 4) : head);
#pragma unroll
            for (int i = 0; i < kBatch; ++i)
              st.step_resolved(static_cast<int>(oc[i]), rc[i], i & 1, kW ? wc[i] : 0.f, kD ? dc[i] : 0.f,
                               R ? xc[i] : 0.f, kP ? pc[i] : 0.f);
          }
          q = nxt;
        }
        if (stop >= nfull) break;
        named_arrive(stop, gate_count(stop));
        stop = stop + 1 < nph ? stop + 1 : nfull;
        }
        if (nfull < nch) {
          const int rem = J - nfull * STEPS;
#pragma unroll
          for (int t = 0; t < STEPS; ++t)
            if (t < rem) st.step(prio_at<1>(q.w, t), t & 1);
        }
      } else if (STREAM) {
        constexpr int STEPS = 32 / PB;  // schedule positions per 256-bit load
        const int nch = (J + STEPS - 1) / STEPS;
        int c = 0, stop = min(arrive_at, nch);  // as above
        for (;;) {
        for (; c < stop; ++c) {
          PrioChunk nxt = q;
          if (c + 1 < nch) nxt = ld_prio32<true>(pg + (c + 1) * 32);
          if ((c + 1) * STEPS <= J) {
#pragma unroll
            for (int t = 0; t < STEPS; ++t) st.step(prio_at<PB>(q.w, t), t & 1);
          } else {
            const int rem = J - c * STEPS;
#pragma unroll
            for (int t = 0; t < STEPS; ++t)
              if (t < rem) st.step(prio_at<PB>(q.w, t), t & 1);
          }
          q = nxt;
        }
        if (stop >= nch) break;
        named_arrive(stop, gate_count(stop));
        stop = stop + 1 < nph ? stop + 1 : nch;
        }
      } else {
        const uint4* prow = reinterpret_cast<const uint4*>(prio_row_s);
        constexpr int STEPS = 16 / PB;  // jobs per 128-bit shared-memory read
        const int nch = (J + STEPS - 1) / STEPS;
        for (int c = 0; c < nch; ++c) {
          const uint4 p = prow[c];
          const uint32_t w[4] = {p.x, p.y, p.z, p.w};
          if ((c + 1) * STEPS <= J) {
#pragma unroll
            for (int t = 0; t < STEPS; ++t) st.step(prio_at<PB>(w, t), t & 1);
          } else {
            const int rem = J - c * STEPS;
#pragma unroll
            for (int t = 0; t < STEPS; ++t)
              if (t < rem) st.step(prio_at<PB>(w, t), t & 1);
          }
        }
      }
      return st.result(a.nodes);
    };
    // SEARCH rounds: score the lane's rows from window `w0` on (warp-uniform).  w0 > 0 resumes from the
    // snapshot taken in front of that window (buffer bit w0-1 of `par`); `save` stores the state in front of
    // every later window into the OTHER buffer (the proposal's boundary states; the caller flips the bits of
    // `par` if it accepts the move).  Snapshot = the 8 sorted slot times + the running score (LaneState::running);
    // a completion parked in `pend` is always folded at a window boundary (even number of steps per window).
    [[maybe_unused]] auto eval_from = [&](const uint8_t* prio_row_s, int w0, uint32_t par, bool save,
                                          float* snap_t) -> float {
      const int J = a.J;
      constexpr int STEPS = 16 / PB;            // schedule positions per 128-bit shared-memory read
      constexpr int CPW = kSnapPos / STEPS;     // reads per window
      const int nch = (J + STEPS - 1) / STEPS;
      if (w0 == 0) {
        st.reset(a.nodes);
      } else {
        const float* sp = snap_t + (((w0 - 1) * 2 + ((par >> (w0 - 1)) & 1u)) * 9) * 32 + lane;
#pragma unroll
        for (int i = 0; i < 8; ++i) st.f[i] = __ldcg(sp + i * 32);
        st.mk = __ldcg(sp + 8 * 32);
        st.pend = 0.f;
      }
      const uint4* prow = reinterpret_cast<const uint4*>(prio_row_s);
      // ONE copy of the unrolled step body in this loop: the kernel is instruction-fetch bound as soon as the
      // hot path spans several unrolled bodies (a window loop around CPW unrolled reads and three inlined call
      // sites stalls on instruction fetch)
#pragma unroll 1
      for (int c = w0 * CPW; c < nch; ++c) {
        if (save && c > w0 * CPW && (c % CPW) == 0) {
          const int b = c / CPW - 1;  // boundary in front of window b + 1
          float* sp = snap_t + ((b * 2 + (((par >> b) & 1u) ^ 1u)) * 9) * 32 + lane;
#pragma unroll
          for (int i = 0; i < 8; ++i) __stcg(sp + i * 32, st.f[i]);
          __stcg(sp + 8 * 32, st.running());
        }
        const uint4 p = prow[c];
        const uint32_t wd[4] = {p.x, p.y, p.z, p.w};
        if ((c + 1) * STEPS <= J) {
#pragma unroll
          for (int t = 0; t < STEPS; ++t) st.step(prio_at<PB>(wd, t), t & 1);
        } else {
          const int rem = J - c * STEPS;
#pragma unroll 1
          for (int t = 0; t < rem; ++t) st.step(PB == 1 ? prio_row_s[c * STEPS + t] : reinterpret_cast<const uint16_t*>(prio_row_s)[c * STEPS + t], -1);
        }
      }
      return st.result(a.nodes);
    };
    if (!SEARCH) {
      float mk = 0.f;
      if (active) {
        mk = evaluate(tile_p + lane * a.row_p);
        a.out[b0 + lane] = mk;
      }
      if (a.best_key != nullptr) fold_best(a.best_key, active, mk, a.id_base + static_cast<uint32_t>(b0 + lane), lane);
      arrive_at = nfull_ch + 1;  // warp 0 opens the stagger barriers in its first tile only
    } else {
      // ---- sf.nrounds Metropolis rounds on the rows of this tile, which stay in shared memory: a rejected
      // move is undone in place, an accepted one writes its few changed bytes through to HBM.  The lane
      // whose candidate lowers the global best key stops moving for the rest of the launch, so that the rows
      // the tail saves (keep_best_tail) are the ones the key was scored on.
      const long long c = cand;
      // lanes beyond the end of the population shadow lane 0's rows (read-only), so that the evaluation below
      // runs converged on valid data in every lane
      const int rl = active ? lane : 0;
      uint8_t* orow_s = tile_o + rl * a.row_o;
      uint8_t* prow_s = tile_p + rl * a.row_p;
      st.orow = orow_s;
      const uint64_t gid = a.sf.chain_base + static_cast<uint64_t>(c);
      float cm = active ? a.sf.cur_mk[c] : 0.f;
      bool moving = active;  // false from the round in which this lane lowers the global best key
      // incremental rounds (one node): boundary snapshots of this tile, filled by one unmodified pass
      const bool inc = !MULTI && a.sf.snap != nullptr;
      const bool win = !MULTI && a.sf.win != 0;
      const int nwin = (a.J + kSnapPos - 1) / kSnapPos;
      float* snap_t = inc ? a.sf.snap + static_cast<size_t>(tile) * (static_cast<size_t>(nwin - 1) * 2 * 9 * 32) : nullptr;
      uint32_t par = 0;  // bit w-1: which buffer holds the current candidate's state in front of window w
      const uint32_t inc_bits = launch_incumbent_bits(a.sf);  // makespan of the incumbent saved before this launch
      // r = -1 (incremental only) is the unmodified pass that fills buffer 0 of every boundary; it shares the
      // one call site of eval_from with the rounds
#pragma unroll 1
      for (int r = inc ? -1 : 0; r < a.sf.nrounds; ++r) {
        const int round = a.sf.round + r;
        const bool fill = r < 0;
        if (!fill && a.sf.resample_every > 0 && round > 1 && (round - 1) % a.sf.resample_every == 0) {
          // tournament inside the warp: take over the rows of a random lane if its candidate is better.
          // Rows move 16 bytes at a time through registers, every lane reading chunk i before any lane
          // writes chunk i, so a lane that is both source and taker is still copied in its old state.
          const uint64_t rr = rng_u64(a.sf.seed ^ 0x7e57a11ull, gid, static_cast<uint64_t>(round));
          const int rival = static_cast<int>(rr >> 59);
          const float rcm = __shfl_sync(0xffffffffu, cm, rival);
          const bool ractive = (__ballot_sync(0xffffffffu, active) >> rival) & 1u;
          const bool take = moving && ractive && rcm < cm;
          const uint4* so = reinterpret_cast<const uint4*>(tile_o + rival * a.row_o);
          const uint4* sp = reinterpret_cast<const uint4*>(tile_p + rival * a.row_p);
          uint4* go = reinterpret_cast<uint4*>(a.sf.cur_o + c * a.stride_o);
          uint4* gp = reinterpret_cast<uint4*>(a.sf.cur_p + c * a.stride_p);
          for (int i = 0; i * 16 < a.copy_o; ++i) {
            const uint4 v = so[i];
            __syncwarp();
            if (take) { reinterpret_cast<uint4*>(orow_s)[i] = v; go[i] = v; }
            __syncwarp();
          }
          for (int i = 0; i * 16 < a.copy_p; ++i) {
            const uint4 v = sp[i];
            __syncwarp();
            if (take) { reinterpret_cast<uint4*>(prow_s)[i] = v; gp[i] = v; }
            __syncwarp();
          }
          if (inc) {
            // ... and its boundary snapshots, from the rival's current buffers into this lane's current buffers.
            // ALL loads of a batch (up to 7 boundaries = 63 words; the evaluation registers are free here) are
            // issued before the first store, so a tournament costs one trip to L2 / HBM per batch, not one per
            // boundary (copying boundary by boundary costs 7 dependent round trips every other round, enough to
            // make incremental scoring slower than scoring from position 0).
            const uint32_t rpar = __shfl_sync(0xffffffffu, par, rival);
            constexpr int kBatch = 7;
            for (int b0s = 0; b0s < nwin - 1; b0s += kBatch) {
              float v[kBatch][9];
#pragma unroll
              for (int bb = 0; bb < kBatch; ++bb) {
                const int b = b0s + bb;
                if (take && b < nwin - 1) {
                  const float* src = snap_t + ((b * 2 + ((rpar >> b) & 1u)) * 9) * 32 + rival;
#pragma unroll
                  for (int i = 0; i < 9; ++i) v[bb][i] = __ldcg(src + i * 32);
                }
              }
              __syncwarp();  // every lane has read its rival's state of this batch before any lane overwrites its own
#pragma unroll
              for (int bb = 0; bb < kBatch; ++bb) {
                const int b = b0s + bb;
                if (take && b < nwin - 1) {
                  float* dst = snap_t + ((b * 2 + ((par >> b) & 1u)) * 9) * 32 + lane;
#pragma unroll
                  for (int i = 0; i < 9; ++i) __stcg(dst + i * 32, v[bb][i]);
                }
              }
              __syncwarp();
            }
          }
          if (take) {
            cm = rcm;
            a.sf.cur_mk[c] = rcm;
          }
        }
        // the window of this round: one draw per (warp's first chain, round), the same in all 32 lanes
        int w0 = 0;
        if (win && !fill) {
          const uint64_t wr = rng_u64(a.sf.seed ^ 0x31d0ull, a.sf.chain_base + static_cast<uint64_t>(a.sf.deal ? tile : b0),
                                      static_cast<uint64_t>(round));
          w0 = draw_window(wr, nwin, a.sf.win_bias);
        }
        Move mv;
        mv.kind = 0; mv.a = mv.b = mv.va = mv.vb = 0;
        if (moving && !fill) {
          if (win) {
            const int p0 = w0 * kSnapPos;
            mv = apply_move_win<PB>(a.sf, round, a.J, gid, orow_s, prow_s, p0, min(kSnapPos, a.J - p0));
          } else {
            mv = apply_move<PB>(a.sf, round, a.J, gid, orow_s, prow_s);
          }
        }
        __syncwarp();  // shadowing lanes read lane 0's rows
        // the one evaluation site: trip 0 is the round's score (resumed from the window's snapshot when
        // incremental), trip 1 — verify hook only — recomputes it from position 0 and compares
        float mk = 0.f;
        const int trips = (inc && !fill && a.sf.verify_bad != nullptr) ? 2 : 1;
#pragma unroll 1
        for (int trip = 0; trip < trips; ++trip) {
          const float got = eval_from(prow_s, (inc && trip == 0) ? w0 : 0, fill ? ~0u : par, inc && trip == 0, snap_t);
          if (trip == 0) mk = got;
          else if (active && __float_as_uint(got) != __float_as_uint(mk)) atomicAdd(a.sf.verify_bad, 1ull);
        }
        if (fill) continue;
        if (moving) {
          bool acc = mk <= cm;
          const float temp = a.sf.temperature[r];
          if (!acc && temp > 0.f && isfinite(mk)) {
            const uint64_t rr = rng_u64(a.sf.seed, gid, 4ull * round + 3);
            const float u = (static_cast<uint32_t>(rr >> 40) + 0.5f) * (1.0f / 16777216.0f);
            acc = u < __expf(-(mk - cm) / temp);
          }
          if (acc) {
            if (mv.kind != 0) {
              write_back<PB>(mv, orow_s, prow_s, a.sf.cur_o + c * a.stride_o, a.sf.cur_p + c * a.stride_p);
              a.sf.cur_mk[c] = mk;
              cm = mk;
              // the boundary states this proposal wrote (windows after w0) are now the current ones
              if (inc) par ^= (w0 + 1 < nwin) ? (~0u << w0) : 0u;
            }
          } else {
            undo_move<PB>(mv, orow_s, prow_s);
            mk = cm;
          }
        }
        if (a.best_key != nullptr) fold_best(a.best_key, active, mk, a.id_base + static_cast<uint32_t>(c), lane);
        if (active && __float_as_uint(mk) < inc_bits) moving = false;  // see launch_incumbent_bits
      }
      st.orow = tile_o + lane * a.row_o;
    }
  }
  if (!tab_ready && threadIdx.x == 0) mbar_wait(bar_tab, 0);  // never leave a bulk copy in flight
  if (kFetch && a.tile_wait != nullptr && lane == 0) {
    atomicAdd(a.tile_wait, t_wait);
    atomicAdd(a.tile_wait + 1, globaltimer_ns() - t_loop);
  }
  if (!SEARCH && fold_pending) try_fold(true);  // before the tail: the publish of this round follows the fold
  if (SEARCH) {
    if (a.sf.keep.counter != nullptr) keep_best_tail(a.sf);
    return;
  }
  if (a.xp.counter != nullptr) {
    // fused exchange: the CTA that finishes last has seen every atomicMin on best_key; it publishes
    // {key, round} in this rank's mailbox (local stores, release at system scope).  Peers read the
    // mailbox over NVLink in k_xchg_reduce (sb_xchg.cu).
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const unsigned done = atomicAdd(a.xp.counter, 1u);
      if (done == gridDim.x - 1) {
        *a.xp.counter = 0;
        __threadfence();
        const unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(a.best_key);
        unsigned long long* slot = a.xp.x.local + (a.xp.seq & 1ull) * 2;
        asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(slot), "l"(k) : "memory");
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(slot + 1), "l"(a.xp.seq) : "memory");
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Generic fallback: any J (prio u8/u16), any row stride; rows are read straight from global
// memory through L1.  The table is staged in shared memory when it fits, else read via L1/L2.
// MULTI keeps the node states in a lane-private shared-memory column as the tile kernel does.
struct GenericArgs {
  const float* tab;
  int J, SG;
  const uint8_t* opt;
  const uint8_t* prio;
  long long B;
  long long stride_o, stride_p;
  float* out;
  unsigned long long* best_key;
  uint32_t id_base;
  int tab_in_smem;
  int nodes;
  int one;
  const float* w;  // obj_weights(OBJ): job weights [J], read with ld.global.nc
  const float* d;  // obj_due(OBJ): job due dates (or tails) [J], likewise
  const float* r;  // R: job release dates [J], likewise
  const float* p;  // obj_penalty(OBJ): job late penalties [J], likewise
  int K;           // obj_scenario(OBJ): the scenario tables at tab, [K][J][SG] (last: the other fields keep their offsets)
  int pad;         // keeps the struct free of implicit padding: a padding hole changes the code of every kernel taking it
};

// One pass of the scenario forms over a candidate's J steps on the table st.tab points to: the batched loop of
// k_eval_generic below, with step_obj(OBJ)'s step (whose kernels keep their own copy of the loop, so that their code
// stays what it was).  The tardiness forms gather the batch's weights and due dates with its runtimes; the makespan
// forms read neither.
template <int PB, Obj OBJ, bool R, class Lane>
__device__ __forceinline__ float generic_pass(Lane& st, const GenericArgs& a, const uint8_t* prow) {
  static_assert(obj_scenario(OBJ), "the scenario forms only");
  constexpr bool kWD = obj_weights(step_obj(OBJ));  // the tardiness step: weights and due dates
  static_assert(kWD == obj_due(step_obj(OBJ)), "a scenario step reads both arrays or neither");
  st.reset(a.nodes);
  constexpr int BATCH = 16;
  int i = 0;
  for (; i + BATCH <= a.J; i += BATCH) {
    int js[BATCH], os[BATCH];
    float rts[BATCH];
    [[maybe_unused]] float xs[BATCH], ws[BATCH], ds[BATCH];
#pragma unroll
    for (int t = 0; t < BATCH; ++t) js[t] = PB == 1 ? prow[i + t] : reinterpret_cast<const uint16_t*>(prow)[i + t];
#pragma unroll
    for (int t = 0; t < BATCH; ++t) os[t] = st.lookup_opt(js[t]);
#pragma unroll
    for (int t = 0; t < BATCH; ++t) rts[t] = st.lookup_rt(js[t], os[t]);
    if constexpr (R) {
#pragma unroll
      for (int t = 0; t < BATCH; ++t) xs[t] = st.lookup_r(js[t]);
    }
    if constexpr (kWD) {
#pragma unroll
      for (int t = 0; t < BATCH; ++t) ws[t] = st.lookup_w(js[t]);
#pragma unroll
      for (int t = 0; t < BATCH; ++t) ds[t] = st.lookup_d(js[t]);
    }
#pragma unroll
    for (int t = 0; t < BATCH; ++t)
      st.step_resolved(os[t], rts[t], t & 1, kWD ? ws[t] : 0.f, kWD ? ds[t] : 0.f, R ? xs[t] : 0.f, 0.f);
  }
  for (; i < a.J; ++i) st.step(PB == 1 ? prow[i] : reinterpret_cast<const uint16_t*>(prow)[i]);
  return st.result(a.nodes);
}

// obj_scenario(OBJ): each lane runs its candidate's J steps once per scenario table, with the makespan form's step,
// and folds the K makespans into the score (scenario_fold); one slot state, whatever K.
template <int PB, bool INT, bool MULTI, Obj OBJ = Obj::Makespan, bool R = false>
__global__ void __launch_bounds__(128) k_eval_generic(const GenericArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr bool kScen = obj_scenario(OBJ);
  const float* tab = a.tab;
  const uint32_t node_bytes = MULTI ? static_cast<uint32_t>(a.nodes) * 1024u : 0u;  // per warp
  float4* node_s = reinterpret_cast<float4*>(smem) + (threadIdx.x >> 5) * (node_bytes / 16);
  if (a.tab_in_smem) {
    float* tab_s = reinterpret_cast<float*>(smem + (blockDim.x >> 5) * node_bytes);
    const int n = kScen ? a.J * a.SG * a.K : a.J * a.SG;
    for (int i = threadIdx.x; i < n; i += blockDim.x) tab_s[i] = a.tab[i];
    __syncthreads();
    tab = tab_s;
  }
  const int lane = threadIdx.x & 31;
  LaneState<INT, MULTI, 0, step_obj(OBJ), 2, R> st;
  st.tab = tab;
  st.wt = a.w;
  st.dd = a.d;
  st.rr = a.r;
  st.pp = a.p;
  st.SG = a.SG;
  st.one = a.one;
  st.ns = node_s + lane;
  const long long nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long Bpad = (a.B + 31) & ~31ll;
  for (long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; b < Bpad; b += nthreads) {
    const bool active = b < a.B;
    float mk = 0.f;
    if (active) {
      st.orow = a.opt + b * a.stride_o;
      const uint8_t* prow = a.prio + b * a.stride_p;
      if constexpr (kScen) {
        for (int k = 0; k < a.K; ++k) {
          st.tab = tab + static_cast<size_t>(k) * a.J * a.SG;
          mk = scenario_fold<OBJ>(mk, generic_pass<PB, OBJ, R>(st, a, prow));
        }
      } else {
      st.reset(a.nodes);
      // batches of 16 positions: 16 independent opt loads, then 16 independent table loads, then the
      // 16 dependent scheduling steps — the global-memory latency is paid once per batch
      constexpr int BATCH = 16;
      int i = 0;
      for (; i + BATCH <= a.J; i += BATCH) {
        int js[BATCH], os[BATCH];
        float rts[BATCH];
#pragma unroll
        for (int t = 0; t < BATCH; ++t) js[t] = PB == 1 ? prow[i + t] : reinterpret_cast<const uint16_t*>(prow)[i + t];
#pragma unroll
        for (int t = 0; t < BATCH; ++t) os[t] = st.lookup_opt(js[t]);
#pragma unroll
        for (int t = 0; t < BATCH; ++t) rts[t] = st.lookup_rt(js[t], os[t]);
        // the batch's release dates, weights, due dates (or tails) and late penalties, gathered with its runtimes
        [[maybe_unused]] float xs[BATCH], ws[BATCH], ds[BATCH], ps[BATCH];
        if constexpr (R) {
#pragma unroll
          for (int t = 0; t < BATCH; ++t) xs[t] = st.lookup_r(js[t]);
        }
        if constexpr (obj_weights(OBJ)) {
#pragma unroll
          for (int t = 0; t < BATCH; ++t) ws[t] = st.lookup_w(js[t]);
        }
        if constexpr (obj_due(OBJ)) {
#pragma unroll
          for (int t = 0; t < BATCH; ++t) ds[t] = st.lookup_d(js[t]);
        }
        if constexpr (obj_penalty(OBJ)) {
#pragma unroll
          for (int t = 0; t < BATCH; ++t) ps[t] = st.lookup_p(js[t]);
        }
#pragma unroll
        for (int t = 0; t < BATCH; ++t)
          st.step_resolved(os[t], rts[t], t & 1, obj_weights(OBJ) ? ws[t] : 0.f, obj_due(OBJ) ? ds[t] : 0.f,
                           R ? xs[t] : 0.f, obj_penalty(OBJ) ? ps[t] : 0.f);
      }
      for (; i < a.J; ++i) st.step(PB == 1 ? prow[i] : reinterpret_cast<const uint16_t*>(prow)[i]);
      mk = st.result(a.nodes);
      }
      a.out[b] = mk;
    }
    if (a.best_key != nullptr) fold_best(a.best_key, active, mk, a.id_base + static_cast<uint32_t>(b), lane);
  }
}

// ------------------------------------------------------------------------------------------
// Slot-exact evaluation: start time and GPU-slot bitmask per job.  The k slots with smallest
// (ready, slot) are found by k ascending scans with a strict '<' (lowest slot wins ties),
// exactly as the oracle states the rule.  Not a throughput kernel: used to decode winners and
// for the slot-index parity tests.  With nodes > 1 the opt byte is (node << 3) | (k - 1), the
// scans run over the job's node only, and the mask is (node << 16) | gpu bits.
struct FullArgs {
  const float* tab;
  int J, SG;
  const uint8_t* opt;
  const uint8_t* prio;
  long long B;
  long long stride_o, stride_p;
  int nodes;
  float* out;
  float* start;         // [B][J] by job, nullable
  uint32_t* slotmask;   // [B][J] by job, nullable
  const float* w;       // obj_weights(OBJ): job weights [J]
  const float* d;       // obj_due(OBJ): job due dates [J] (TailMakespan: the delivery tails)
  const float* r;       // R: job release dates [J] (ceiled with INT)
  const float* p;       // obj_penalty(OBJ): job late penalties [J]
  int K;                // obj_scenario(OBJ): the scenario tables at tab, [K][J][SG] (last: the other fields keep their
                        // offsets); `start` (nullable) then receives every scenario's makespan, [B][K]
  int pad;              // keeps the struct free of implicit padding: a padding hole changes the code of every kernel
                        // taking it
};

// The score is folded here on its own, not through ls_step: this kernel is the library's slot-exact cross-check of
// the fast kernels, so it restates every objective's fold (in the same fp32 operations).
template <int PB, bool INT, Obj OBJ = Obj::Makespan, bool R = false>
__global__ void __launch_bounds__(128) k_eval_full(const FullArgs a);

// obj_scenario(OBJ): the slot-exact score of each scenario table, the makespan M_k or the tardiness form's total S_k
// (start times and slot masks are not written: the host takes them from the makespan form on the nominal table), into
// a.start ([B][K]), folded into the score in scenario order
template <int PB, bool INT, Obj OBJ, bool R>
__device__ __forceinline__ void eval_full_scenarios(const FullArgs& a) {
  const long long nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
  const bool multi = a.nodes > 1;
  for (long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; b < a.B; b += nthreads) {
    const uint8_t* orow = a.opt + b * a.stride_o;
    const uint8_t* prow = a.prio + b * a.stride_p;
    float score = 0.f;
    for (int sc = 0; sc < a.K; ++sc) {
      const float* tab = a.tab + static_cast<size_t>(sc) * a.J * a.SG;
      float ready[kMaxNodes * kSlots];
      for (int g = 0; g < a.nodes * kSlots; ++g) ready[g] = 0.f;
      float mk = 0.f;
      for (int i = 0; i < a.J; ++i) {
        const int j = PB == 1 ? prow[i] : reinterpret_cast<const uint16_t*>(prow)[i];
        const int o = orow[j];
        const int k = (o & 7) + 1;
        const int node = multi ? (o >> 3) : 0;
        const float rt = __ldg(tab + static_cast<size_t>(j) * a.SG + (multi ? (o & 7) : o));
        float* rd = ready + node * kSlots;
        uint32_t taken = 0;
        float s = 0.f;
        for (int q = 0; q < k; ++q) {
          int best = -1;
          float bv = 0.f;
          for (int g = 0; g < kSlots; ++g) {
            const bool free_slot = ((taken >> g) & 1u) == 0u;
            if (free_slot && (best < 0 || rd[g] < bv)) {
              best = g;
              bv = rd[g];
            }
          }
          taken |= 1u << best;
          s = bv;
        }
        if constexpr (R) s = fmaxf(s, __ldg(a.r + j));
        const float hold = (INT && isfinite(rt)) ? ceilf(rt) : rt;
        const float nxt = s + hold;
        for (int g = 0; g < kSlots; ++g)
          if ((taken >> g) & 1u) rd[g] = nxt;
        if constexpr (step_obj(OBJ) == Obj::Tardiness)
          mk = __fadd_rn(mk, __fmul_rn(__ldg(a.w + j), fmaxf(__fsub_rn(s + rt, __ldg(a.d + j)), 0.f)));
        else
          mk = fmaxf(mk, s + rt);
      }
      if (a.start) a.start[b * a.K + sc] = mk;
      score = scenario_fold<OBJ>(score, mk);
    }
    if (a.out) a.out[b] = score;
  }
}

template <int PB, bool INT, Obj OBJ, bool R>
__global__ void __launch_bounds__(128) k_eval_full(const FullArgs a) {
  if constexpr (obj_scenario(OBJ)) {
    eval_full_scenarios<PB, INT, OBJ, R>(a);
    return;
  } else {
  const long long nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
  const bool multi = a.nodes > 1;
  for (long long b = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; b < a.B; b += nthreads) {
    const uint8_t* orow = a.opt + b * a.stride_o;
    const uint8_t* prow = a.prio + b * a.stride_p;
    float ready[kMaxNodes * kSlots];
    for (int g = 0; g < a.nodes * kSlots; ++g) ready[g] = 0.f;
    float mk = 0.f;
    for (int i = 0; i < a.J; ++i) {
      const int j = PB == 1 ? prow[i] : reinterpret_cast<const uint16_t*>(prow)[i];
      const int o = orow[j];
      const int k = (o & 7) + 1;
      const int node = multi ? (o >> 3) : 0;
      const float rt = __ldg(a.tab + static_cast<size_t>(j) * a.SG + (multi ? (o & 7) : o));
      float* rd = ready + node * kSlots;
      uint32_t taken = 0;
      float s = 0.f;
      for (int q = 0; q < k; ++q) {
        int best = -1;
        float bv = 0.f;
        for (int g = 0; g < kSlots; ++g) {
          const bool free_slot = ((taken >> g) & 1u) == 0u;
          if (free_slot && (best < 0 || rd[g] < bv)) {
            best = g;
            bv = rd[g];
          }
        }
        taken |= 1u << best;
        s = bv;  // scans return non-decreasing values: the last one is the k-th smallest
      }
      if constexpr (R) s = fmaxf(s, __ldg(a.r + j));  // ls_step<..., kRelease>: not before the release
      const float hold = (INT && isfinite(rt)) ? ceilf(rt) : rt;
      const float nxt = s + hold;
      for (int g = 0; g < kSlots; ++g)
        if ((taken >> g) & 1u) rd[g] = nxt;
      if constexpr (OBJ == Obj::TailMakespan)
        mk = fmaxf(mk, __fadd_rn(s + rt, __ldg(a.d + j)));
      else if constexpr (OBJ == Obj::LateCount)  // +inf once a job has no runtime (LaneState::result)
        mk = isinf(s + rt) ? INFINITY : __fadd_rn(mk, __fmul_rn(__ldg(a.w + j), s + rt > __ldg(a.d + j) ? 1.f : 0.f));
      else if constexpr (OBJ == Obj::MaxTardiness)
        mk = fmaxf(mk, __fmul_rn(__ldg(a.w + j), fmaxf(__fsub_rn(s + rt, __ldg(a.d + j)), 0.f)));
      else if constexpr (OBJ == Obj::Tardiness)
        mk = __fadd_rn(mk, __fmul_rn(__ldg(a.w + j), fmaxf(__fsub_rn(s + rt, __ldg(a.d + j)), 0.f)));
      else if constexpr (OBJ == Obj::SquaredTardiness) {
        const float t = fmaxf(__fsub_rn(s + rt, __ldg(a.d + j)), 0.f);
        mk = __fadd_rn(mk, __fmul_rn(__ldg(a.w + j), __fmul_rn(t, t)));
      }
      else if constexpr (OBJ == Obj::LatePenalty) {
        const float x = __fsub_rn(s + rt, __ldg(a.d + j));
        mk = __fadd_rn(mk, x > 0.f ? __fadd_rn(__ldg(a.p + j), __fmul_rn(__ldg(a.w + j), x)) : 0.f);
      }
      else if constexpr (OBJ == Obj::CompletionPenalty) {
        float t = __fmul_rn(__ldg(a.w + j), s + rt);
        if (s + rt > __ldg(a.d + j)) t = __fadd_rn(t, __ldg(a.p + j));
        mk = __fadd_rn(mk, t);
      }
      else if constexpr (OBJ == Obj::WeightedSum) mk = __fadd_rn(mk, __fmul_rn(__ldg(a.w + j), s + rt));
      else if constexpr (OBJ == Obj::Sum) mk = mk + (s + rt);  // the left fold in schedule order
      else mk = fmaxf(mk, s + rt);
      if (a.start) a.start[b * a.J + j] = s;
      if (a.slotmask) a.slotmask[b * a.J + j] = (static_cast<uint32_t>(node) << 16) | taken;
    }
    if (a.out) a.out[b] = mk;
  }
  }
}

// ------------------------------------------------------------------------------------------
// validation of external candidates: prio rows are permutations of 0..J-1 and every opt byte
// names an existing (finite) table cell (and, with several nodes, an existing node).
// bad[0] counts offending rows.
__global__ void k_validate(const float* tab, int J, int SG, int nodes, const uint8_t* opt, const uint8_t* prio, int pb,
                           long long B, long long stride_o, long long stride_p, unsigned long long* bad, int by_pos) {
  const int lane = threadIdx.x & 31;
  const long long warp = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  extern __shared__ uint32_t seen_all[];
  const int words = (J + 31) / 32;
  uint32_t* seen = seen_all + (threadIdx.x >> 5) * words;
  for (long long b = warp; b < B; b += nwarps) {
    for (int w = lane; w < words; w += 32) seen[w] = 0;
    __syncwarp();
    bool ok = true;
    const uint8_t* orow = opt + b * stride_o;
    const uint8_t* prow = prio + b * stride_p;
    for (int i = lane; i < J; i += 32) {
      const int j = pb == 1 ? prow[i] : reinterpret_cast<const uint16_t*>(prow)[i];
      if (j >= J) {
        ok = false;
      } else {
        const uint32_t old = atomicOr(&seen[j >> 5], 1u << (j & 31));
        if (old & (1u << (j & 31))) ok = false;
      }
      int o = orow[i];  // the option of job i — or, by_pos, of the job scheduled i-th
      if (nodes > 1) {
        if ((o >> 3) >= nodes) ok = false;
        o &= 7;
      }
      const int job = by_pos ? (j < J ? j : 0) : i;
      if (o >= SG || !isfinite(tab[static_cast<size_t>(job) * SG + o])) ok = false;
    }
    ok = __all_sync(0xffffffffu, ok);
    if (!ok && lane == 0) atomicAdd(bad, 1ull);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------ host side
static int round_row(int bytes) {
  int r16 = (bytes + 15) / 16;
  if ((r16 & 1) == 0) r16 += 1;  // odd multiple of 16 B -> conflict-free per-lane 128-bit reads
  return r16 * 16;
}

int plan_tiles(const Device& dev, int J, int SG, int pb, bool stream, int nodes, TilePlan* tp, bool tab_global,
               int arrays) {
  tp->row_o = round_row(J);
  tp->row_p = round_row(J * pb);
  tp->copy_o = (J + 15) & ~15;
  tp->copy_p = (J * pb + 15) & ~15;
  size_t tab_bytes = tab_global ? 0 : ((static_cast<size_t>(J) * SG * 4 + 15) & ~size_t(15));
  if (!tab_global) tab_bytes += arrays * job_array_bytes(J);
  const size_t per_warp = 32u * static_cast<size_t>(tp->row_o + (stream ? 0 : tp->row_p)) +
                          (nodes > 1 ? static_cast<size_t>(nodes) * 1024u : 0u);
  int nw = stream ? 16 : 12;  // block size limits: 512 / 384 threads (128 registers per thread)
  while (nw > 0 && tab_bytes + 16 * ((1 + nw + 1) / 2) + nw * per_warp > dev.smem_optin) --nw;
  tp->warps = nw;
  tp->smem = tab_bytes + (((1 + nw) * 8 + 15) & ~15) + nw * per_warp;
  return nw;
}

using TileKernel = void (*)(TileArgs);

// both row buffers start on 16-byte boundaries and stay on them from row to row: TMA bulk copies can fetch the rows
static bool bulk_aligned(const EvalCall& c) {
  return (c.stride_o % 16 == 0) && (c.stride_p % 16 == 0) && (reinterpret_cast<uintptr_t>(c.opt) % 16 == 0) &&
         (reinterpret_cast<uintptr_t>(c.prio) % 16 == 0);
}

// the fields of TileArgs that the call and the tile plan fix
static TileArgs tile_args(const EvalCall& c, const TilePlan& tp) {
  TileArgs a;
  a.tab = c.tab; a.J = c.J; a.SG = c.SG; a.opt = c.opt; a.prio = c.prio; a.B = c.B;
  a.stride_o = c.stride_o; a.stride_p = c.stride_p;
  a.row_o = tp.row_o; a.row_p = tp.row_p; a.copy_o = tp.copy_o; a.copy_p = tp.copy_p;
  a.nodes = c.nodes;
  a.out = c.out; a.best_key = c.best_key; a.id_base = c.id_base;
  a.w = c.w;
  a.d = c.d;
  a.r = c.r;
  a.p = c.p;
  a.ntiles = (c.B + 31) / 32;
  a.one = 1;
  a.packed = a.stagger = 0;
  a.tile_wait = nullptr;
  return a;
}

static cudaError_t launch_tiles(const Device& dev, TileKernel kern, const TileArgs& a, const TilePlan& tp,
                                cudaStream_t st) {
  long long ctas = (a.ntiles + tp.warps - 1) / tp.warps;
  int grid = static_cast<int>(ctas < dev.sm_count ? ctas : dev.sm_count);
  return launch(kern, grid, tp.warps * 32, tp.smem, st, a);
}

cudaError_t eval_launch(const Device& dev, const EvalCall& c, cudaStream_t st, int* path_used) {
  if (c.B <= 0) return cudaSuccess;
  const int pb = c.J <= 256 ? 1 : 2;
  const bool multi = c.nodes > 1;
  const bool bulk_ok = bulk_aligned(c);
  const bool stream_ok = bulk_ok && (c.stride_p % 32 == 0) && (reinterpret_cast<uintptr_t>(c.prio) % 32 == 0) &&
                         !(c.flags & HOOK_NO_STREAM);
  const int arrays = job_arrays(c.obj, c.flags);
  TilePlan tp;
  int nw = 0;
  bool stream = false, tabg = false;
  const bool scen = obj_scenario(c.obj);  // the tile kernels have no scenario forms: the generic kernel scores them
  if (!c.force_generic && !scen) {
    if (stream_ok) {
      nw = plan_tiles(dev, c.J, c.SG, pb, true, c.nodes, &tp, false, arrays);
      stream = nw >= 2 && c.stride_o >= tp.copy_o && c.stride_p >= ((c.J * pb + 31) & ~31);
      if (!stream && !multi) {
        // the table itself does not fit beside the tiles: keep it in global memory
        nw = plan_tiles(dev, c.J, c.SG, pb, true, c.nodes, &tp, true);
        stream = tabg = nw >= 2 && c.stride_o >= tp.copy_o && c.stride_p >= ((c.J * pb + 31) & ~31);
      }
    }
    if (!stream) nw = plan_tiles(dev, c.J, c.SG, pb, false, c.nodes, &tp, false, arrays);
  }
  if (nw >= 2) {
    TileArgs a = tile_args(c, tp);
    a.use_bulk = stream || (bulk_ok && (c.stride_o >= tp.copy_o) && (c.stride_p >= tp.copy_p));
    a.xp = c.xp;
    if (path_used) *path_used = tabg ? 4 : (stream ? 3 : (a.use_bulk ? 2 : 1));
    // the headline shape (u8 priorities streamed, one node, table in shared memory): address arithmetic on the FMA
    // pipe unless HOOK_PLAIN_ADDR asks for the plain form
    const bool fma_addr = pb == 1 && stream && !tabg && !multi && !(c.flags & HOOK_PLAIN_ADDR);
    if (stream && !tabg && !multi) {  // the tile-boundary measures of k_eval_tiles (kFetch)
      a.packed = c.stride_o == tp.copy_o && c.stride_p == tp.copy_p && !(c.tile_debug & TILE_DEBUG_ROW_COPIES);
      if (a.packed) a.row_o = tp.copy_o;
      a.stagger = !(c.tile_debug & TILE_DEBUG_NO_STAGGER);
      a.tile_wait = c.tile_wait;
    }
    const TileKernel kern = with_eval_types(pb, c.flags, c.obj, [&](auto PB, auto INT, auto OBJ, auto R) -> TileKernel {
      if (tabg) return k_eval_tiles<PB, INT, true, false, false, true, 0, OBJ, R>;
      if constexpr (PB == 1) {
        if (fma_addr) return k_eval_tiles<1, INT, true, false, false, false, 1, OBJ, R>;
      }
      return with_bool(stream, [&](auto STREAM) {
        return with_bool(multi, [&](auto MULTI) -> TileKernel {
          return k_eval_tiles<PB, INT, STREAM, MULTI, false, false, 0, OBJ, R>;
        });
      });
    });
    return launch_tiles(dev, kern, a, tp, st);
  }
  GenericArgs g;
  g.tab = c.tab; g.J = c.J; g.SG = c.SG; g.opt = c.opt; g.prio = c.prio; g.B = c.B;
  g.stride_o = c.stride_o; g.stride_p = c.stride_p; g.out = c.out; g.best_key = c.best_key;
  g.id_base = c.id_base; g.tab_in_smem = 0; g.nodes = c.nodes; g.one = 1; g.w = c.w; g.d = c.d; g.r = c.r;
  g.p = c.p;
  g.K = c.K;
  g.pad = 0;
  if (path_used) *path_used = 0;
  // the scenario tables always fit (check_per_job holds them to scenario_smem, which asks for more than this)
  const size_t tab_bytes = static_cast<size_t>(c.J) * c.SG * 4 * (scen ? c.K : 1);
  size_t smem = multi ? static_cast<size_t>(4) * c.nodes * 1024u : 0u;  // 4 warps per CTA
  if (tab_bytes <= dev.smem_optin / 2 || scen) {
    g.tab_in_smem = 1;
    smem += tab_bytes;
  }
  long long blocks = (c.B + 127) / 128;
  long long cap = static_cast<long long>(dev.sm_count) * 8;
  int grid = static_cast<int>(blocks < cap ? blocks : cap);
  if (grid < 1) grid = 1;
  using GenericKernel = void (*)(GenericArgs);
  const auto pick = [&](auto PB, auto INT, auto OBJ, auto R) -> GenericKernel {
    return with_bool(multi, [&](auto MULTI) -> GenericKernel { return k_eval_generic<PB, INT, MULTI, OBJ, R>; });
  };
  const GenericKernel kern = scen ? with_scenario_types(pb, c.flags, c.obj, pick) : with_eval_types(pb, c.flags, c.obj, pick);
  return launch(kern, grid, 128, smem, st, g);
}

// 2 = both rows of a candidate fit in shared memory for at least 8 warps: the tile kernel runs the fused
// round (all moves); 0 = they do not: the search keeps a position-major population (sb_search.cu: 16 warps
// at any J, where only a few tile warps would fit) or, when even the table does not fit, runs unfused rounds
int search_round_mode(const Device& dev, int J, int SG, int nodes, int arrays) {
  const int pb = J <= 256 ? 1 : 2;
  TilePlan tp;
  return plan_tiles(dev, J, SG, pb, false, nodes, &tp, false, arrays) >= 8 ? 2 : 0;
}

// One fused search round over `c.B` chains whose current candidates are (c.opt, c.prio).  Returns
// cudaErrorNotSupported when the shared-memory tiles (both rows resident, >= 4 warps) do not fit;
// the caller then runs the unfused propose / evaluate / accept round.
cudaError_t search_round_launch(const Device& dev, const EvalCall& c, const SearchFuse& sf, cudaStream_t st) {
  if (c.B <= 0) return cudaSuccess;
  const int pb = c.J <= 256 ? 1 : 2;
  TilePlan tp;
  const int arrays = job_arrays(c.obj, c.flags);
  if (search_round_mode(dev, c.J, c.SG, c.nodes, arrays) == 0 || !bulk_aligned(c)) return cudaErrorNotSupported;
  plan_tiles(dev, c.J, c.SG, pb, false, c.nodes, &tp, false, arrays);
  if (c.stride_o < tp.copy_o || c.stride_p < tp.copy_p) return cudaErrorNotSupported;
  TileArgs a = tile_args(c, tp);
  a.use_bulk = 1;
  a.sf = sf;
  const TileKernel kern = with_eval_types(pb, c.flags, c.obj, [&](auto PB, auto INT, auto OBJ, auto R) {
    return with_bool(c.nodes > 1, [&](auto MULTI) -> TileKernel {
      return k_eval_tiles<PB, INT, false, MULTI, true, false, 0, OBJ, R>;
    });
  });
  return launch_tiles(dev, kern, a, tp, st);
}

cudaError_t eval_full_launch(const Device& dev, const EvalCall& c, float* start, uint32_t* slotmask, cudaStream_t st) {
  if (c.B <= 0) return cudaSuccess;
  const int pb = c.J <= 256 ? 1 : 2;
  FullArgs a;
  a.tab = c.tab; a.J = c.J; a.SG = c.SG; a.opt = c.opt; a.prio = c.prio; a.B = c.B;
  a.stride_o = c.stride_o; a.stride_p = c.stride_p; a.nodes = c.nodes < 1 ? 1 : c.nodes;
  a.out = c.out; a.start = start; a.slotmask = slotmask; a.w = c.w; a.d = c.d; a.r = c.r;
  a.p = c.p;
  a.K = c.K;
  a.pad = 0;
  long long blocks = (c.B + 127) / 128;
  long long cap = static_cast<long long>(dev.sm_count) * 16;
  int grid = static_cast<int>(blocks < cap ? blocks : cap);
  using FullKernel = void (*)(FullArgs);
  const auto pick = [](auto PB, auto INT, auto OBJ, auto R) -> FullKernel { return k_eval_full<PB, INT, OBJ, R>; };
  if (obj_scenario(c.obj)) return cudaErrorInvalidValue;  // eval_full_scenarios_launch
  return launch(with_eval_types(pb, c.flags, c.obj, pick), grid, 128, 0, st, a);
}

cudaError_t eval_full_scenarios_launch(const Device& dev, const EvalCall& c, float* mks, cudaStream_t st) {
  if (c.B <= 0) return cudaSuccess;
  if (!obj_scenario(c.obj)) return cudaErrorInvalidValue;
  const int pb = c.J <= 256 ? 1 : 2;
  FullArgs a = {};
  a.tab = c.tab; a.J = c.J; a.SG = c.SG; a.opt = c.opt; a.prio = c.prio; a.B = c.B;
  a.stride_o = c.stride_o; a.stride_p = c.stride_p; a.nodes = c.nodes < 1 ? 1 : c.nodes;
  a.out = c.out; a.r = c.r; a.w = c.w; a.d = c.d;
  a.K = c.K;
  a.start = mks;
  long long blocks = (c.B + 127) / 128;
  long long cap = static_cast<long long>(dev.sm_count) * 16;
  int grid = static_cast<int>(blocks < cap ? blocks : cap);
  using FullKernel = void (*)(FullArgs);
  const auto pick = [](auto PB, auto INT, auto OBJ, auto R) -> FullKernel { return k_eval_full<PB, INT, OBJ, R>; };
  return launch(with_scenario_types(pb, c.flags, c.obj, pick), grid, 128, 0, st, a);
}

cudaError_t validate_launch(const Device& dev, const EvalCall& c, unsigned long long* bad, cudaStream_t st, bool by_pos) {
  if (c.B <= 0) return cudaSuccess;
  const int pb = c.J <= 256 ? 1 : 2;
  const int words = (c.J + 31) / 32;
  const int threads = 128;
  size_t smem = static_cast<size_t>(threads / 32) * words * 4;
  long long blocks = (c.B + 3) / 4;
  long long cap = static_cast<long long>(dev.sm_count) * 8;
  int grid = static_cast<int>(blocks < cap ? blocks : cap);
  k_validate<<<grid, threads, smem, st>>>(c.tab, c.J, c.SG, c.nodes, c.opt, c.prio, pb, c.B, c.stride_o, c.stride_p, bad,
                                          by_pos ? 1 : 0);
  return cudaGetLastError();
}

}  // namespace sb
