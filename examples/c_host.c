/* A plain-C host of the drop-in boundary (include/saturn_b200.h): what a non-Python caller of the
 * reference's solver would link against.  It plans J synthetic training jobs on one node of 8 GPUs:
 *
 *   sb_create -> sb_set_table (T[J][S][G], the profiler's table) -> sb_search_run (replaces
 *   prob.solve(), milp.py:321-327) -> sb_decode (replaces reading the MILP variables, milp.py:330-352)
 *
 * Build:  gcc -O2 -Iinclude examples/c_host.c -Lsaturn_b200 -lsaturn_b200 -Wl,-rpath,$PWD/saturn_b200 -lm -o c_host
 * Run:    ./c_host [J] [seed]          (prints the plan; needs an H100)
 * Output is line-oriented so that tests/test_gpu_solver.py can re-score the plan with the CPU oracle. */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "saturn_b200.h"

#define CHECK(call)                                                         \
  do {                                                                      \
    int rc__ = (call);                                                      \
    if (rc__ != 0) {                                                        \
      fprintf(stderr, "%s failed (%d): %s\n", #call, rc__, sb_last_error()); \
      return 1;                                                             \
    }                                                                       \
  } while (0)

static uint64_t lcg(uint64_t* s) {
  *s = *s * 6364136223846793005ull + 1442695040888963407ull;
  return *s >> 33;
}

int main(int argc, char** argv) {
  const int J = argc > 1 ? atoi(argv[1]) : 24;
  uint64_t seed = argc > 2 ? (uint64_t)atoll(argv[2]) : 7;
  const int S = 2, G = 8;
  if (J < 1 || J > 4096) return 2;

  /* T[j][s][g]: runtime of job j under strategy s on g+1 GPUs */
  float* T = (float*)malloc(sizeof(float) * J * S * G);
  uint8_t gcount[8];
  for (int g = 0; g < G; ++g) gcount[g] = (uint8_t)(g + 1);
  for (int j = 0; j < J; ++j) {
    const double base = 600.0 + (double)(lcg(&seed) % 30000);
    for (int s = 0; s < S; ++s) {
      const double alpha = 0.55 + 0.4 * (double)(lcg(&seed) % 1000) / 1000.0;
      for (int g = 0; g < G; ++g) T[(j * S + s) * G + g] = (float)(base * (1.0 + 0.2 * s) / pow(g + 1.0, alpha));
    }
  }
  printf("J %d S %d G %d\n", J, S, G);
  printf("T");
  for (int i = 0; i < J * S * G; ++i) printf(" %.9g", T[i]);
  printf("\n");

  sb_handle* h = NULL;
  CHECK(sb_create(0, NULL, &h));
  CHECK(sb_set_table(h, T, gcount, J, S, G, 1));

  int64_t wave = 0;
  CHECK(sb_search_wave(h, SB_FLAG_REDUCED, &wave));
  sb_search_params p = {0};
  p.seed = 1;
  p.chains = wave;
  p.flags = SB_FLAG_INTEGER_STARTS | SB_FLAG_REDUCED;
  p.t_start = 5e-4f;
  p.t_end = 1e-6f;
  sb_search_control c = {0};
  c.rounds = 200;
  c.resample_every = 4;
  c.sync_every = 16;
  c.patience = 64;
  c.heuristic_seeds = 1;
  c.time_budget_s = 5.0;

  uint8_t* opt = (uint8_t*)malloc(J);
  uint16_t* prio16 = (uint16_t*)malloc(sizeof(uint16_t) * J);
  uint8_t* prio8 = (uint8_t*)prio16; /* u8 priorities when J <= 256 */
  sb_search_result res;
  CHECK(sb_search_run(h, &p, &c, NULL, NULL, opt, prio16, &res));

  float* start = (float*)malloc(sizeof(float) * J);
  uint32_t* mask = (uint32_t*)malloc(sizeof(uint32_t) * J);
  uint8_t* strat = (uint8_t*)malloc(J);
  uint8_t* gpus = (uint8_t*)malloc(J);
  float mk = 0.f;
  CHECK(sb_decode(h, opt, prio16, p.flags, start, mask, strat, gpus, NULL, &mk));

  printf("makespan %.9g search %.9g candidates %lld rounds %d stop %d wall_ms %.3f\n", mk, res.makespan,
         (long long)res.evaluated, res.rounds, res.stop_reason, res.wall_s * 1e3);
  printf("opt");
  for (int j = 0; j < J; ++j) printf(" %d", opt[j]);
  printf("\nprio");
  for (int i = 0; i < J; ++i) printf(" %d", J <= 256 ? prio8[i] : prio16[i]);
  printf("\n");
  for (int j = 0; j < J; ++j)
    printf("job %d strategy %d gpus %d start %.0f mask 0x%02x\n", j, strat[j], gpus[j], start[j], mask[j] & 0xff);

  CHECK(sb_destroy(h));
  free(T); free(opt); free(prio16); free(start); free(mask); free(strat); free(gpus);
  return 0;
}
