// sb_search.h — device-resident state of one search population.
#pragma once
#include "sb_internal.h"

namespace sb {

struct SearchDev {
  int J = 0, pb = 1;
  int nodes = 1;  // > 1: opt bytes carry the node in bits 3..
  int pos = 0;    // 1: the population stores opt BY POSITION (large J, see sb_search.cu)
  long long chains = 0;
  uint64_t chain_base = 0;
  uint64_t seed = 0;
  long long stride_o = 0, stride_p = 0;  // bytes, multiples of 16
  uint8_t *cur_o = nullptr, *cur_p = nullptr, *prop_o = nullptr, *prop_p = nullptr;
  float *cur_mk = nullptr, *prop_mk = nullptr;
  const uint8_t* vopt = nullptr;  // [J][8]
  const int* nvalid = nullptr;    // [J]
  // [0] best key of this population, [1] key of the saved encoding; equal after every call (k_keep_best saves
  // the rows of [0]'s chain, so [0] must never name a chain that has moved on since it was scored)
  unsigned long long* keys = nullptr;
  uint8_t *best_o = nullptr, *best_p = nullptr;
};

cudaError_t search_init_population(const SearchDev& s, cudaStream_t st);
cudaError_t search_propose(const SearchDev& s, int round, cudaStream_t st);
cudaError_t search_keep_best(const SearchDev& s, bool from_cur, cudaStream_t st);
cudaError_t search_accept(const SearchDev& s, int round, float temperature, cudaStream_t st);
cudaError_t search_init_population_pos(const SearchDev& s, cudaStream_t st);
size_t search_pos_smem(int J, int SG, int nodes, int warps, int arrays = 0);  // arrays: job_arrays(obj, flags)
// w: the job weights [J] (obj_weights(obj)), else nullptr; d: the due dates or tails [J] (obj_due(obj)); r: the
// release dates [J] (SB_FLAG_RELEASE; ceiled with SB_FLAG_INTEGER_STARTS); K: obj_scenario(obj), the number of scenario
// tables at tab ([K][J][SG])
cudaError_t search_pos_launch(const Device& dev, const SearchDev& s, const float* tab, const float* w, const float* d,
                              const float* r, const float* p, int SG, unsigned flags, Obj obj, long long first,
                              long long count, bool eval_only, const SearchFuse& sf, cudaStream_t st, int tab_home = 0,
                              int K = 0);
int eval_pos_home(const Device& dev, int J, int SG, int nodes, unsigned flags, Obj obj, int K = 0);
cudaError_t eval_pos_launch(const Device& dev, const EvalCall& c, cudaStream_t st, int* path = nullptr);
cudaError_t opt_by_position_launch(const Device& dev, const EvalCall& c, uint8_t* out, cudaStream_t st);
cudaError_t search_resample(const SearchDev& s, int round, cudaStream_t st);
cudaError_t search_inject(const SearchDev& s, const uint8_t* cand_o, const uint8_t* cand_p, long long first,
                          int copies, cudaStream_t st);

}  // namespace sb
