/* CPU ORACLE (test infrastructure — NOT product code).
 *
 * The worst and mean total (weighted) tardiness over runtime scenarios (oracle/ref_scenario_tardiness.py) in plain C,
 * fp32, with OpenMP over candidates, in one pass: scenario k's runtime of job j is fl32(f[k][j] * tab[j][...]), the
 * schedule on it is the release-date rule of oracle/ref_release.c (each job takes the k slots with smallest
 * (ready, slot) of its node, ties to the lowest slot, and holds them until start + ceil(rt) under integer starts or
 * start + rt, with start = max(largest ready time among them, r[j])), and S_k is the left fold from +0 in schedule
 * order of fl(w_j * max(fl(C_j - d_j), 0)), each add rounded.  The score is max_k S_k (objective 0) or the left fold
 * acc = acc + S_k from +0 in scenario order (objective 1).  r is given as the schedule uses it (ceiled under integer
 * starts, all zero without release dates), w and d as fp32, by the Python side (unit weights, d = 0 for the completion
 * forms).  Built with -ffp-contract=off.
 *
 * Encodings (include/saturn_b200.h): tab[J][S][8] runtimes (+inf = absent), opt[j] = (s << 3) | (k - 1) or, with
 * several nodes, (node << 3) | (k - 1) on the reduced table (S = 1), prio[i] = job scheduled i-th, f[K][J].
 *
 * Build: gcc -O2 -fopenmp -shared -fPIC -ffp-contract=off oracle/ref_scenario_tardiness.c \
 *            -o oracle/libref_scenario_tardiness.so
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#define NSLOT 8
#define NODES_MAX 8

static float total_one(const float* tab, int J, int S, const float* f, const uint8_t* opt, const uint8_t* prio,
                       int prio_bytes, int integer_starts, int nodes, const float* r, const float* w, const float* d) {
  float ready_all[NODES_MAX * NSLOT];
  int order[NSLOT];
  float acc = 0.f;
  for (int g = 0; g < NODES_MAX * NSLOT; ++g) ready_all[g] = 0.f;
  for (int i = 0; i < J; ++i) {
    int j = prio_bytes == 1 ? prio[i] : ((const uint16_t*)prio)[i];
    int o = opt[j];
    int k = (o & 7) + 1;
    int node = nodes > 1 ? (o >> 3) : 0;
    if (node >= nodes) return INFINITY;
    float rt = f[j] * tab[(size_t)j * S * 8 + (nodes > 1 ? (o & 7) : o)];
    float* ready = ready_all + node * NSLOT;
    for (int g = 0; g < NSLOT; ++g) {
      int q = g;
      while (q > 0 && ready[order[q - 1]] > ready[g]) { order[q] = order[q - 1]; --q; }
      order[q] = g;
    }
    float s = ready[order[k - 1]];
    if (r[j] > s) s = r[j];
    float hold = (integer_starts && isfinite(rt)) ? ceilf(rt) : rt;
    float nxt = s + hold;
    for (int c = 0; c < k; ++c) ready[order[c]] = nxt;
    float e = s + rt;
    float late = e - d[j];
    float t = late > 0.f ? late : 0.f;
    float term = w[j] * t;
    acc = acc + term;
  }
  return acc;
}

int ref_scenario_tardiness_f32(const float* tab, int J, int S, const float* f, int K, const uint8_t* opt,
                               const void* prio, int prio_bytes, int64_t B, int integer_starts, int nodes,
                               const float* r, const float* w, const float* d, int objective, float* score,
                               float* Sk, int nthreads) {
  if (J <= 0 || S <= 0 || K < 1 || K > 8) return -1;
  if (nodes < 1 || nodes > NODES_MAX || (nodes > 1 && S != 1)) return -3;
  if (prio_bytes != 1 && prio_bytes != 2) return -2;
  if (objective != 0 && objective != 1) return -4;
#pragma omp parallel for schedule(dynamic, 64) num_threads(nthreads > 0 ? nthreads : 1)
  for (int64_t b = 0; b < B; ++b) {
    const uint8_t* ob = opt + (size_t)b * J;
    const uint8_t* pb = (const uint8_t*)prio + (size_t)b * J * prio_bytes;
    float acc = 0.f;
    for (int k = 0; k < K; ++k) {
      float m = total_one(tab, J, S, f + (size_t)k * J, ob, pb, prio_bytes, integer_starts, nodes, r, w, d);
      if (Sk) Sk[(size_t)b * K + k] = m;
      if (objective == 0) acc = m > acc ? m : acc;
      else acc = acc + m;
    }
    score[b] = acc;
  }
  return 0;
}
