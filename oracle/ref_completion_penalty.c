/* CPU ORACLE (test infrastructure — NOT product code).
 *
 * The completion penalty of list schedules (oracle/ref_completion_penalty.py) in plain C with OpenMP over
 * candidates.  The schedule is the release-date rule of oracle/ref_release.c: each job takes the k slots with smallest
 * (ready, slot) of its node (ties to the lowest slot) and holds them until start + ceil(rt) (integer_starts) or
 * start + rt, with start = max(largest ready time among them, r[j]); r is given as the schedule uses it (ceiled under
 * integer starts, all zero without release dates, by the Python side).  The score is the left fold in schedule order
 *     e = start + rt,  t = w[j] * e,  t = e > d[j] ? t + p[j] : t,  acc = acc + t  from +0,
 * every step rounded on its own (w all ones for unit weights).  A job with no runtime (rt = +inf) gives a +inf term,
 * so the candidate scores +inf with no special case.  Built with -ffp-contract=off.
 *
 * Encodings (include/saturn_b200.h): tab[J][S][8] runtimes (+inf = absent), opt[j] = (s << 3) | (k - 1) or, with
 * several nodes, (node << 3) | (k - 1) on the reduced table (S = 1), prio[i] = job scheduled i-th.
 *
 * Build: gcc -O2 -fopenmp -shared -fPIC -ffp-contract=off oracle/ref_completion_penalty.c
 *            -o oracle/libref_completion_penalty.so
 */
#include <math.h>
#include <stdint.h>
#include <stddef.h>

#define NSLOT_MAX 8
#define NODES_MAX 8

#define DEFINE_CP(NAME, REAL, CEIL)                                                          \
  static void NAME##_one(const REAL* tab, int J, int S, const uint8_t* opt,                  \
                         const uint8_t* prio, int prio_bytes, int integer_starts,            \
                         int nslot, int nodes, const REAL* w, const REAL* d, const REAL* r,  \
                         const REAL* p, REAL* total, REAL* start_out, uint32_t* mask_out) {  \
    REAL ready_all[NODES_MAX * NSLOT_MAX];                                                   \
    int order[NSLOT_MAX];                                                                    \
    REAL acc = 0;                                                                            \
    int bad = 0;                                                                             \
    for (int g = 0; g < NODES_MAX * NSLOT_MAX; ++g) ready_all[g] = 0;                        \
    for (int i = 0; i < J; ++i) {                                                            \
      int j = prio_bytes == 1 ? prio[i] : ((const uint16_t*)prio)[i];                        \
      int o = opt[j];                                                                        \
      int k = (o & 7) + 1;                                                                   \
      int node = nodes > 1 ? (o >> 3) : 0;                                                   \
      REAL rt = tab[(size_t)j * S * 8 + (nodes > 1 ? (o & 7) : o)];                          \
      if (k > nslot || node >= nodes) { bad = 1; break; }                                    \
      REAL* ready = ready_all + node * NSLOT_MAX;                                            \
      for (int g = 0; g < nslot; ++g) {                                                      \
        int q = g;                                                                           \
        while (q > 0 && ready[order[q - 1]] > ready[g]) { order[q] = order[q - 1]; --q; }    \
        order[q] = g;                                                                        \
      }                                                                                      \
      REAL s = ready[order[k - 1]];                                                          \
      if (r[j] > s) s = r[j];                                                                \
      REAL hold = (integer_starts && isfinite(rt)) ? CEIL(rt) : rt;                          \
      REAL nxt = s + hold;                                                                   \
      uint32_t m = 0;                                                                        \
      for (int c = 0; c < k; ++c) { ready[order[c]] = nxt; m |= 1u << order[c]; }           \
      if (start_out) start_out[j] = s;                                                       \
      if (mask_out) mask_out[j] = ((uint32_t)node << 16) | m;                                \
      REAL e = s + rt;                                                                       \
      REAL t = w[j] * e;                                                                     \
      if (e > d[j]) t = t + p[j];                                                            \
      acc = acc + t;                                                                         \
    }                                                                                        \
    *total = bad ? (REAL)INFINITY : acc;                                                     \
  }                                                                                          \
  int NAME(const REAL* tab, int J, int S, const uint8_t* opt, const void* prio,              \
           int prio_bytes, int64_t B, int integer_starts, int nslot, int nodes,              \
           const REAL* w, const REAL* d, const REAL* r, const REAL* p, REAL* total,          \
           REAL* start_out, uint32_t* mask_out, int nthreads) {                              \
    if (J <= 0 || S <= 0 || nslot < 1 || nslot > NSLOT_MAX) return -1;                       \
    if (nodes < 1 || nodes > NODES_MAX || (nodes > 1 && S != 1)) return -3;                  \
    if (prio_bytes != 1 && prio_bytes != 2) return -2;                                       \
    if (!w || !d || !r || !p) return -4;                                                     \
    _Pragma("omp parallel for schedule(dynamic, 64) num_threads(nthreads > 0 ? nthreads : 1)") \
    for (int64_t b = 0; b < B; ++b)                                                          \
      NAME##_one(tab, J, S, opt + (size_t)b * J, (const uint8_t*)prio +                      \
                 (size_t)b * J * prio_bytes, prio_bytes, integer_starts, nslot, nodes, w, d, \
                 r, p, total + b, start_out ? start_out + (size_t)b * J : 0,                 \
                 mask_out ? mask_out + (size_t)b * J : 0);                                   \
    return 0;                                                                                \
  }

DEFINE_CP(ref_completion_penalty_f32, float, ceilf)
DEFINE_CP(ref_completion_penalty_f64, double, ceil)
