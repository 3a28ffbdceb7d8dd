/* saturn_b200.h — C ABI of the H100-native SPASE solver hot path.
 *
 * This is the drop-in boundary for the ONE path of knagrecha/saturn that this
 * repository accelerates: `saturn.solver.solve()` (reference
 * saturn/solver/milp.py:23-445), whose arithmetic the reference delegates to a
 * third-party MILP binary (PuLP -> Gurobi/CBC, milp.py:321-327).  The library
 * replaces that solver call with a parallel search over list-schedule
 * candidates evaluated by hand-written sm_90a CUDA kernels.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch / Python types.
 *   - every function returns 0 on success, a negative sb_status on failure;
 *     sb_last_error() returns a thread-local human-readable message.
 *   - the caller allocates every buffer; the library never frees caller memory.
 *   - "device pointer" = memory on the handle's CUDA device (e.g.
 *     torch.Tensor.data_ptr()).  Functions ending in _host take host pointers
 *     and perform the copies themselves.
 *   - one handle is single-threaded; separate handles are independent.
 *   - no CPU fallback exists: without a CUDA device sb_create fails with
 *     SB_ERR_CUDA.
 *
 * Encodings (shared with the oracle, oracle/ref_eval.py)
 *   T[J][S][G]   fp32, row-major: runtime in seconds of job j under strategy s
 *                on gcount[g] GPUs — the profiled table the reference stores in
 *                Task.strategies (saturn/core/representations/Task.py:118,
 *                produced by saturn/trial_runner/PerformanceEvaluator.py:96-115).
 *   opt[b][j]    uint8: (s << 3) | (k - 1), k = GPU count of job j's option.
 *   prio[b][i]   uint8 (J <= 256) or uint16: job scheduled i-th; each row is a
 *                permutation of 0..J-1.
 *   rows of opt / prio are `row_stride` ELEMENTS apart (>= J), and BOTH buffers must span
 *   B * row_stride elements (the last row included: the aligned paths fetch whole 16- / 32-byte
 *   chunks of every row, and sb_eval_host copies B * row_stride elements per buffer).  Rows that are
 *   32-byte aligned (base pointers and byte strides multiples of 32) take the
 *   fast path (TMA bulk copies + 32-byte streaming loads); 16-byte aligned rows
 *   use TMA bulk copies only; anything else is fetched with plain loads.
 *
 * Evaluation rule (one node, 8 GPU slots; reference milp.py:62,139-149,209-319)
 *   ready[0..8) = 0
 *   for i in 0..J-1: j = prio[i]; k = (opt[j] & 7) + 1; rt = T(j, opt[j])
 *       sel   = k slots with smallest (ready, slot)      (ties -> lowest slot)
 *       start = max(ready[sel])
 *       ready[sel] = start + (integer_starts ? ceil(rt) : rt)
 *   makespan = max_j (start_j + rt_j)
 * With SB_FLAG_SUM_COMPLETION the score is the sum of completion times instead:
 *   total = sum_j (start_j + rt_j), in fp32 a left fold in schedule order, acc = acc + (start + rt) from +0
 * (one add per job, never paired or reassociated; the oracle folds the same way and agrees bit for bit).
 * With SB_FLAG_WEIGHTED as well (per-job weights w_j > 0, sb_set_weights) it is the weighted sum:
 *   total = sum_j w_j (start_j + rt_j), acc = acc + (w_j * (start_j + rt_j)) from +0 in schedule order, with TWO
 * fp32 roundings per job (the product, then the sum; never one fused multiply-add).  w = 1 gives exactly the
 * unweighted fold, w = 2 exactly twice it (barring overflow).
 * With SB_FLAG_DUE as well (per-job due dates d_j, sb_set_due; unit weights unless SB_FLAG_WEIGHTED) it is the
 * weighted tardiness:
 *   total = sum_j w_j max(0, start_j + rt_j - d_j), from +0 in schedule order per job: e = start + rt (as above),
 *   l = e - d, t = max(l, +0), acc = acc + (w * t), every step rounded on its own (no fused or reassociated step).
 * d = 0 gives exactly the weighted fold, due dates at or past every completion give +0, w = 2 exactly twice w = 1.
 * The score is >= +0, so the (bits << 32) | id key still orders by it.
 * With SB_FLAG_LATE_COUNT as well it is the (weighted) number of late jobs instead:
 *   total = sum_j w_j [start_j + rt_j > d_j], from +0 in schedule order per job: e = start + rt (as above),
 *   acc = acc + (e > d ? w : +0), one rounding per job.  A job that completes exactly at its due date is on time.
 * Unit weights give the exact count; integer weights with sum_j w_j < 2^24 give an exact sum in any order.  Due dates
 * at or past every completion give +0, due dates below every completion give sum_j w_j, w = 2 exactly twice w = 1.
 * The comparison is made in fp32 on the fp32 due date, so a completion within rounding of a fractional due date is
 * decided as the tardiness fold decides it.  A candidate that gives a job an option it does not have (rt = +inf)
 * scores +inf, as under every other objective, though the fold alone would add only that job's weight.
 * With SB_FLAG_MAX_TARDINESS instead it is the maximum weighted tardiness:
 *   score = max_j w_j max(0, start_j + rt_j - d_j), from +0 in schedule order per job: e = start + rt, l = e - d,
 *   t = max(l, +0), x = w * t (each rounded on its own, the tardiness fold's term bit for bit), acc = max(acc, x).
 * d = 0 with unit weights gives exactly the makespan, due dates at or past every completion give +0, w = 2 exactly
 * twice w = 1 (barring overflow).  The score is >= +0.  A job with no runtime (rt = +inf) gives a +inf term, so the
 * candidate scores +inf without a special case.  w_j = 1 / p*_j and d_j = max(r_j, 0), with p*_j a lower bound on
 * job j's runtime, make it the maximum stretch (slowdown) of the jobs, max_j (C_j - max(r_j, 0)) / p*_j.
 * With SB_FLAG_SQUARED instead it is the (weighted) squared tardiness:
 *   total = sum_j w_j max(0, start_j + rt_j - d_j)^2, from +0 in schedule order per job: e = start + rt, l = e - d,
 *   t = max(l, +0) (the tardiness fold's t bit for bit), u = t * t, x = w * u, acc = acc + x, every step rounded on
 *   its own (no fused multiply-add).
 * Due dates at or past every completion give +0, w = 2 exactly twice w = 1 (barring overflow).  The score is >= +0.  A
 * job with no runtime (rt = +inf) gives a +inf term.  d_j = max(r_j, 0) makes it the squared flow time
 * sum_j w_j (C_j - max(r_j, 0))^2 (sum_j w_j C_j^2 without release dates).
 * With SB_FLAG_LATE_PENALTY as well (per-job late penalties p_j >= 0, sb_set_penalty) it is the late penalty:
 *   total = sum_j [C_j > d_j] (p_j + w_j (C_j - d_j)), from +0 in schedule order per job: e = start + rt, x = e - d,
 *   then acc = acc + (x > 0 ? p + (w * x) : +0), the product and the sum each rounded on their own (no fused
 *   multiply-add).
 * A job that completes exactly at its due date is on time.  p = 0 gives exactly the tardiness fold of SB_FLAG_DUE,
 * due dates at or past every completion give +0, and the score is >= +0.  A job with no runtime (rt = +inf) gives a
 * +inf term.  The comparison C > d is made in fp32, as the late count makes it.
 * With SB_FLAG_COMPLETION_PENALTY instead (penalties from sb_set_penalty as well) it is the completion penalty:
 *   total = sum_j (w_j C_j + [C_j > d_j] p_j), from +0 in schedule order per job: e = start + rt, t = w * e, then
 *   t = t + p when e > d, then acc = acc + t, every step rounded on its own (no fused multiply-add).
 * p = 0 gives exactly the weighted completion fold (the unweighted sum without SB_FLAG_WEIGHTED).  A job that
 * completes exactly at its due date is on time; a job with no runtime (rt = +inf) gives a +inf term.  One due date H
 * for every job with every p above any sum_j w_j C_j makes it min sum_j w_j C_j subject to makespan <= H.
 * The schedule, every start and every slot mask are the same under every objective.
 * With SB_FLAG_MAX_LATENESS (per-job due dates d_j, sb_set_due) the score is the maximum lateness
 * L_max = max_j (start_j + rt_j - d_j), emitted as the tail makespan L_max + D >= +0 with D = max_t d_t:
 *   q_j = D - d_j (>= +0, made once in fp32 by sb_set_due), e = start + rt (as above), x = e + q (one rounding),
 *   score = max_j x, a max fold from +0 like the makespan's.
 * Every score the library emits then holds L_max + D, so the key still orders by it; subtract D to get L_max.  Due
 * dates shifted by one constant give the same q, hence the same scores and plans.  d = c for a constant c gives
 * exactly the makespan.
 * With SB_FLAG_RELEASE (per-job release dates r_j, sb_set_release; valid under every objective above) a job may not
 * start before its release:
 *       start = max(max(ready[sel]), r_j)
 * slot selection and everything after the start are unchanged, and so is every score's fold.  r <= 0 means the job
 * is already released (max(ready, r) = ready, since ready >= +0).  With integer_starts the release enters as
 * ceil(r_j), so every start stays an integer.  All-zero release dates give exactly the results without the flag.
 * With integer_starts the slot state is the integer time a slot becomes usable, start + ceil(rt);
 * SURVEY.md §8a writes the same rule as `start = ceil(max ready)` over real-valued ready times.  Starts,
 * makespans and the set of k slots taken are identical (ceil is monotone); the one observable difference
 * is WHICH of several slots that become free within the same integer second is taken first: here ties are
 * between equal integer usable-times and go to the lowest slot index.  The oracle (oracle/ref_eval.py)
 * defines the rule the tests hold the kernels to.
 */
#ifndef SATURN_B200_H
#define SATURN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_ABI_VERSION 1
#define SB_NSLOT 8          /* GPUs per node, reference milp.py:62 */
#define SB_MAX_STRATEGIES 32 /* 5 strategy bits in an opt byte */
#define SB_MAX_NODES 8       /* multi-node tables: up to 8 nodes x 8 GPUs */

typedef enum sb_status {
  SB_OK = 0,
  SB_ERR_ARG = -1,       /* bad argument */
  SB_ERR_CUDA = -2,      /* CUDA runtime / driver error, no device */
  SB_ERR_STATE = -3,     /* call out of order (e.g. eval before set_table) */
  SB_ERR_UNSUPPORTED = -4,
  SB_ERR_NOMEM = -5
} sb_status;

/* flags for sb_eval* / sb_search */
#define SB_FLAG_INTEGER_STARTS 1u /* MILP start variables are Integer, milp.py:142-143 */
#define SB_FLAG_REDUCED 2u        /* opt bytes carry s = 0; the min-over-strategies table is used
                                     (PerformanceEvaluator.py:101-115) */
#define SB_FLAG_OPT_BY_POSITION 4u /* sb_eval only: opt[b][i] is the option of the job scheduled i-th (= of job
                                    * prio[b][i]) instead of the option of job i.  Both rows are then consumed in
                                    * order and stream through registers: no shared-memory tile, full occupancy
                                    * at any J.  Needs 32-byte aligned rows.  A one-node table beyond one SM's
                                    * shared memory (C5 with all 8 strategies: 256 KB) is read through L1 / L2. */
#define SB_FLAG_POST_KEY 8u       /* sb_eval: when the last candidate is scored, publish *best_key in this
                                     rank's peer-visible mailbox (see sb_xchg_*); the same kernel does both */
#define SB_FLAG_FOLD_PREV 16u     /* with SB_FLAG_POST_KEY: the kernel's prologue first MINs into *best_key the keys
                                     all ranks published in the PREVIOUS round (one-round pipelined exchange:
                                     the NVLink latency hides under the evaluation); finish with sb_xchg_reduce */
#define SB_FLAG_ALT_WARPSCAN 32u   /* sb_eval only, one node: score with the ALTERNATE kernel shape — a candidate's 8
                                     slot times spread over 8 lanes and combined with warp shuffles (the shape
                                     BASELINE.json's north_star sketches), 4 candidates per warp.  Same results;
                                     kept to be measured against the shipped lane-per-candidate kernel
                                     (bench.py configs.C4_alt_shape), not to be used. */
#define SB_FLAG_SUM_COMPLETION 64u /* objective = sum of completion times (the mean job completion time x J) instead of
                                     the makespan.  Accepted by sb_eval, sb_eval_host, sb_eval_full, sb_decode and the
                                     search (sb_search_params.flags).  EVERY score the library emits then holds that
                                     sum: makespan_out, sb_decode's makespan, the packed best keys (a non-negative
                                     fp32, so the key is still an arg-min), sb_search_best's and
                                     sb_search_result's makespan, the history; sb_search_control.target_makespan
                                     then targets the sum.  Starts and slot masks do not change.  The search's
                                     temperature unit becomes the incumbent's MEAN completion (sum / J), and
                                     sb_search_seed_lpt plants shortest-processing-time orders.  Not available with
                                     SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_WEIGHTED 128u      /* with SB_FLAG_SUM_COMPLETION only (else SB_ERR_ARG), after sb_set_weights (else
                                     SB_ERR_STATE): the objective is the WEIGHTED sum of completion times
                                     sum_j w_j (start_j + rt_j) (see the evaluation rule above).  Accepted wherever
                                     SB_FLAG_SUM_COMPLETION is, sb_search_run_multi included (every handle must hold
                                     weights); every score the library emits then holds the weighted sum.  The
                                     search's temperature unit becomes the incumbent's weighted sum / sum_j w_j, and
                                     sb_search_seed_lpt plants WSPT orders (Smith's rule: ascending rt / w, ties by
                                     job index).  Not available with SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_DUE 256u           /* with SB_FLAG_SUM_COMPLETION only (else SB_ERR_ARG), after sb_set_due (else
                                     SB_ERR_STATE): the objective is the total tardiness against the due dates,
                                     weighted by the weights with SB_FLAG_WEIGHTED as well (see the evaluation rule
                                     above).  Accepted wherever SB_FLAG_WEIGHTED is, sb_search_run_multi included
                                     (every handle must hold due dates); every score the library emits then holds
                                     the tardiness.  The search's temperature unit becomes max(incumbent / sum_j w_j,
                                     sum_j w_j min_k rt_jk / sum_j w_j) (the second term: the weighted mean of each
                                     job's smallest proposable runtime), sb_search_run stops as soon as the
                                     incumbent is +0 (stop_reason 3), and sb_search_seed_lpt plants EDD orders
                                     (ascending due date, ties by runtime / weight, then job index).  Not available
                                     with SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_RELEASE 512u       /* after sb_set_release (else SB_ERR_STATE): no job starts before its release date
                                     (see the evaluation rule above).  Valid under every objective (the makespan,
                                     SB_FLAG_SUM_COMPLETION, SB_FLAG_WEIGHTED and SB_FLAG_DUE), and accepted by
                                     sb_eval, sb_eval_host, sb_eval_full, sb_decode and the search,
                                     sb_search_run_multi included (every handle must hold release dates).  The
                                     search's temperature unit and stopping rules are unchanged; sb_search_seed_lpt
                                     re-sorts each seed's order stably by ascending release date (ceiled with
                                     SB_FLAG_INTEGER_STARTS), so jobs released together keep the objective's order.
                                     Not available with SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_MAX_LATENESS 1024u /* after sb_set_due (else SB_ERR_STATE): the objective is the maximum lateness,
                                     scored as the tail makespan L_max + max_t d_t (see the evaluation rule above).
                                     Not combinable with SB_FLAG_SUM_COMPLETION, SB_FLAG_WEIGHTED or SB_FLAG_DUE, and
                                     refused when max d - min d >= 2^24 (SB_ERR_ARG both).  Below that spread the
                                     tails of integer due dates are exact; fractional due dates get q rounded to
                                     fp32 like any fp32 subtraction (the device and the oracle round alike).
                                     Valid with SB_FLAG_RELEASE and several nodes; accepted wherever SB_FLAG_DUE is,
                                     sb_search_run_multi included (every handle must hold due dates).  The search's
                                     temperature unit is the makespan's (a fraction of the incumbent score), it has
                                     no stop at zero (stop_reason 3 only follows target_makespan, which then targets
                                     the tail makespan), and sb_search_seed_lpt plants the unit-weight EDD orders of
                                     SB_FLAG_DUE.  Not available with SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_LATE_COUNT 2048u   /* with SB_FLAG_SUM_COMPLETION | SB_FLAG_DUE only (SB_FLAG_WEIGHTED optional; else
                                     SB_ERR_ARG, as with SB_FLAG_MAX_LATENESS): the objective is the (weighted)
                                     number of late jobs, sum_j w_j [C_j > d_j], instead of their tardiness (see the
                                     evaluation rule above).  It reads the weights and due dates of SB_FLAG_DUE and
                                     needs nothing else.  Accepted by sb_eval, sb_eval_host, sb_eval_full, sb_decode
                                     and the search, sb_search_run_multi included; every score the library emits
                                     then holds the count, and target_makespan targets it.  The search's temperature
                                     unit becomes sum_j w_j (the count of all jobs with unit weights), it stops as
                                     soon as the incumbent is +0 (stop_reason 3), and sb_search_seed_lpt plants the
                                     EDD orders of SB_FLAG_DUE repaired by Moore-Hodgson's rule: while the list
                                     schedule of the on-time sequence has a late job, the job with the largest
                                     k * rt / w up to and including the first late one (the later on ties) moves to
                                     the back, where the moved jobs keep their EDD order.  Not available with
                                     SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_MAX_TARDINESS 4096u /* with SB_FLAG_SUM_COMPLETION | SB_FLAG_DUE only (SB_FLAG_WEIGHTED optional; else
                                     SB_ERR_ARG), and not with SB_FLAG_LATE_COUNT or SB_FLAG_MAX_LATENESS (SB_ERR_ARG):
                                     the tardiness terms are folded with max instead of +, and the objective is the
                                     maximum (weighted) tardiness max_j w_j max(0, C_j - d_j) (see the evaluation
                                     rule above).  It reads the weights and due dates of SB_FLAG_DUE and needs
                                     nothing else.  Accepted by sb_eval, sb_eval_host, sb_eval_full, sb_decode and
                                     the search, sb_search_run_multi included; every score the library emits then
                                     holds the maximum, and target_makespan targets it.  The search's temperature
                                     unit becomes max(incumbent, max_j w_j min_k rt_jk) (a max, not divided by
                                     sum_j w_j), it stops as soon as the incumbent is +0 (stop_reason 3), and
                                     sb_search_seed_lpt plants the EDD orders of SB_FLAG_DUE.  Not available with
                                     SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_SQUARED 8192u      /* with SB_FLAG_SUM_COMPLETION | SB_FLAG_DUE only (SB_FLAG_WEIGHTED optional; else
                                     SB_ERR_ARG), and not with SB_FLAG_LATE_COUNT, SB_FLAG_MAX_TARDINESS or
                                     SB_FLAG_MAX_LATENESS (SB_ERR_ARG): each tardiness is squared before it is
                                     weighted, and the objective is the (weighted) squared tardiness
                                     sum_j w_j max(0, C_j - d_j)^2 (see the evaluation rule above).  It reads the
                                     weights and due dates of SB_FLAG_DUE and needs nothing else.  With
                                     SB_FLAG_WEIGHTED it is SB_ERR_ARG unless J * max_j w_j * 2^50 < FLT_MAX
                                     (recorded by sb_set_weights): a tardiness below 2^25 squares below 2^50, so
                                     below that bound the sum cannot overflow to +inf.  Accepted by sb_eval,
                                     sb_eval_host, sb_eval_full, sb_decode and the search, sb_search_run_multi
                                     included; every score the library emits then holds the sum of squares, and
                                     target_makespan targets it.  The search's temperature unit becomes
                                     max(incumbent / sum_j w_j, sum_j w_j (min_k rt_jk)^2 / sum_j w_j) (SB_FLAG_DUE's
                                     floor with each runtime squared), it stops as soon as the incumbent is +0
                                     (stop_reason 3), and sb_search_seed_lpt plants the EDD orders of SB_FLAG_DUE.
                                     Not available with SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_LATE_PENALTY 16384u /* with SB_FLAG_SUM_COMPLETION | SB_FLAG_DUE only (SB_FLAG_WEIGHTED, the rate per
                                     unit of time late, optional; else SB_ERR_ARG), and not with SB_FLAG_LATE_COUNT,
                                     SB_FLAG_MAX_TARDINESS, SB_FLAG_SQUARED or SB_FLAG_MAX_LATENESS (SB_ERR_ARG),
                                     after sb_set_penalty (else SB_ERR_STATE, checked after the due dates and before
                                     the release dates): each late job adds its fixed penalty to its weighted
                                     tardiness, and the objective is sum_j [C_j > d_j] (p_j + w_j (C_j - d_j)) (see
                                     the evaluation rule above).  Accepted by sb_eval, sb_eval_host, sb_eval_full,
                                     sb_decode and the search, sb_search_run_multi included (every handle must hold
                                     penalties); every score the library emits then holds the total penalty, and
                                     target_makespan targets it.  The search's temperature unit becomes
                                     max(incumbent / sum_j w_j, (sum_j w_j min_k rt_jk + sum_j p_j) / sum_j w_j)
                                     (SB_FLAG_DUE's floor with the penalties added), it stops as soon as the
                                     incumbent is +0 (stop_reason 3), and sb_search_seed_lpt plants the EDD orders of
                                     SB_FLAG_DUE.  Not available with SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_COMPLETION_PENALTY 32768u /* with SB_FLAG_SUM_COMPLETION | SB_FLAG_DUE only (SB_FLAG_WEIGHTED optional;
                                     else SB_ERR_ARG), and not with SB_FLAG_LATE_PENALTY, SB_FLAG_LATE_COUNT,
                                     SB_FLAG_MAX_TARDINESS, SB_FLAG_SQUARED or SB_FLAG_MAX_LATENESS (SB_ERR_ARG), after
                                     sb_set_penalty (else SB_ERR_STATE, checked after the due dates and before the
                                     release dates): the (weighted) completion time plus a fixed penalty for each
                                     missed due date, sum_j (w_j C_j + [C_j > d_j] p_j) (see the evaluation rule
                                     above).  Accepted wherever SB_FLAG_LATE_PENALTY is; every score the library emits
                                     then holds that total, and target_makespan targets it.  The search's temperature
                                     unit is the completion unit (incumbent / sum_j w_j, no sum of penalties added),
                                     it does not stop at 0, and sb_search_seed_lpt plants the completion orders (SPT,
                                     WSPT with SB_FLAG_WEIGHTED), not the EDD orders of SB_FLAG_DUE.  Not available
                                     with SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_WORST_MAKESPAN 65536u /* after sb_set_scenarios (else SB_ERR_STATE): the objective is the worst makespan
                                     over the K runtime scenarios, max_k M_k, where M_k is the makespan of the same
                                     candidate (options and order, the list rule re-run) on scenario table k,
                                     T_k[j][c] = fp32(f[k][j] * T[j][c]).  Not combinable with SB_FLAG_MEAN_MAKESPAN,
                                     SB_FLAG_SUM_COMPLETION, SB_FLAG_WEIGHTED, SB_FLAG_DUE, SB_FLAG_MAX_LATENESS,
                                     SB_FLAG_LATE_COUNT, SB_FLAG_MAX_TARDINESS, SB_FLAG_SQUARED, SB_FLAG_LATE_PENALTY or
                                     SB_FLAG_COMPLETION_PENALTY (SB_ERR_ARG); valid with SB_FLAG_RELEASE and several
                                     nodes.  The K tables must fit in one CTA's shared memory beside the release dates
                                     and the node states (else SB_ERR_UNSUPPORTED).  Accepted by sb_eval, sb_eval_host,
                                     sb_eval_full, sb_eval_scenarios, sb_decode and the search, sb_search_run_multi
                                     included; sb_eval_full and sb_decode report the start times and GPU slots of the
                                     nominal schedule (on T).  The search runs without incremental rounds, with the
                                     makespan's temperature unit (the incumbent's score) and seeds.  Not available with
                                     SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_MEAN_MAKESPAN 131072u /* as SB_FLAG_WORST_MAKESPAN, but the score is the sum of the K makespans, the
                                     left fold acc = acc + M_k (fp32, each add rounded) in scenario order from +0: K
                                     times the mean makespan, with the same arg-min. */
#define SB_FLAG_WORST_TARDINESS 262144u /* modifies SB_FLAG_SUM_COMPLETION | SB_FLAG_DUE [| SB_FLAG_WEIGHTED], after
                                     sb_set_scenarios (else SB_ERR_STATE): the objective is the worst total (weighted)
                                     tardiness over the K runtime scenarios, max_k S_k, where S_k is the tardiness
                                     form's score, the left fold from +0 in schedule order of
                                     fp32(w_j * max(C_jk - d_j, 0)) (each add rounded), of the same candidate (options
                                     and order, the list rule re-run) on scenario table k.  Not the largest per-job
                                     tardiness (that is SB_FLAG_MAX_TARDINESS).  With every d = +0 the score is the worst
                                     (weighted) sum of completion times bit for bit.  Without SB_FLAG_SUM_COMPLETION |
                                     SB_FLAG_DUE, with SB_FLAG_MEAN_TARDINESS, SB_FLAG_LATE_COUNT,
                                     SB_FLAG_MAX_TARDINESS, SB_FLAG_SQUARED, SB_FLAG_LATE_PENALTY,
                                     SB_FLAG_COMPLETION_PENALTY, SB_FLAG_MAX_LATENESS, SB_FLAG_WORST_MAKESPAN or
                                     SB_FLAG_MEAN_MAKESPAN it is SB_ERR_ARG; valid with SB_FLAG_RELEASE and several
                                     nodes.  The K tables, the weights and the due dates must fit in one CTA's shared
                                     memory beside the release dates and the node states (else SB_ERR_UNSUPPORTED).
                                     Accepted where SB_FLAG_WORST_MAKESPAN is, with the same routes; sb_eval_full and
                                     sb_decode report the start times and GPU slots of the nominal schedule (on T).  The
                                     search runs without incremental rounds, plants the EDD seeds of SB_FLAG_DUE on the
                                     nominal table, stops at a score of 0, and takes the tardiness form's temperature
                                     unit.  Not available with SB_FLAG_ALT_WARPSCAN (SB_ERR_UNSUPPORTED). */
#define SB_FLAG_MEAN_TARDINESS 524288u /* as SB_FLAG_WORST_TARDINESS, but the score is the sum of the K totals, the
                                     left fold acc = acc + S_k (fp32, each add rounded) in scenario order from +0: K
                                     times the mean total tardiness, with the same arg-min; the search's temperature
                                     floor is K times the tardiness form's. */
#define SB_IPC_HANDLE_BYTES 64

typedef struct sb_handle sb_handle;

/* ---- lifecycle -------------------------------------------------------------------------- */
int sb_abi_version(void);
const char* sb_last_error(void);
/* device: CUDA ordinal.  stream: the cudaStream_t every call on this handle is queued on (NULL = the
 * context's default stream, which is what PyTorch uses unless told otherwise).  Work is ordered
 * with the caller's other work on that stream; nothing synchronises unless documented. */
int sb_create(int device, void* stream, sb_handle** out);
int sb_destroy(sb_handle* h);
/* blocks until everything queued on the handle's stream is done */
int sb_sync(sb_handle* h);

/* ---- the table (replaces milp.py:77-81 building gpu_time_tuples) --------------------------
 * T: host or device pointer, fp32 [J][S][G]; gcount: host pointer, uint8 [G], values 1..8.
 * nodes: 1..SB_MAX_NODES nodes of 8 GPUs (the reference takes len(ray.nodes()), milp.py:58-62).  A
 * task runs on exactly one node and its gang takes GPUs of that node only (milp.py:117-137,209-227).
 * With nodes > 1 candidates are evaluated on the reduced table only (SB_FLAG_REDUCED) and the opt
 * byte reads (node << 3) | (k - 1).  Builds on the device: the canonical table
 * tab[J][S][8] (column k-1, +inf where no option), and the min-over-strategies table
 * tmin[J][8] with argS[J][8] (first minimum wins, PerformanceEvaluator.py:105-110).
 * Every cell must be >= 0 (-0.0 counts as zero), +inf or a sentinel: a negative or NaN cell returns SB_ERR_ARG (the
 * list-scheduling step cannot score a negative hold, and a NaN would read as an absent option).  T may be device
 * memory, so the cells are checked on the device while the table is built.  After that refusal, as after a failed
 * build, the handle has no table (sb_eval and the rest return SB_ERR_STATE until a table is set). */
int sb_set_table(sb_handle* h, const float* T, const uint8_t* gcount, int J, int S, int G, int nodes);
/* Runtime threshold at and above which a table cell counts as one of the profiler's sentinels
 * (1e6 "not profiled", 1e8 "failed", PerformanceEvaluator.py:99,106) and is never PROPOSED by the
 * search (it is still evaluated like any number if a caller's candidate selects it).  Default 1e6;
 * pass +inf to treat every finite cell as usable.  Takes effect at the next sb_set_table. */
int sb_set_sentinel(sb_handle* h, float threshold);
/* Per-job weights for SB_FLAG_WEIGHTED: w host fp32 [J], every value finite and > 0 (else SB_ERR_ARG, as is a J
 * that differs from the table's); w = NULL clears them.  SB_ERR_STATE before sb_set_table.  sb_set_table clears
 * the weights; setting or clearing them ends the current search (sb_search_init again). */
int sb_set_weights(sb_handle* h, const float* w, int J);
/* Per-job due dates for SB_FLAG_DUE and SB_FLAG_MAX_LATENESS: d host fp32 [J] in the runtimes' units from the plan's
 * t = 0, every value
 * finite with |d| < 2^24 (negative: already overdue) (else SB_ERR_ARG, as is a J that differs from the table's);
 * d = NULL clears them.  SB_ERR_STATE before sb_set_table.  sb_set_table clears the due dates; setting or clearing
 * them ends the current search (sb_search_init again).  It also makes the delivery tails max_t d_t - d_j that
 * SB_FLAG_MAX_LATENESS scores, once, and records whether max d - min d < 2^24 (else that flag is refused). */
int sb_set_due(sb_handle* h, const float* d, int J);
/* Per-job release dates for SB_FLAG_RELEASE: r host fp32 [J] in the runtimes' units from the plan's t = 0, every
 * value finite with |r| < 2^24 (r <= 0: already released) (else SB_ERR_ARG, as is a J that differs from the
 * table's); r = NULL clears them.  SB_ERR_STATE before sb_set_table.  The ceiled copy that SB_FLAG_INTEGER_STARTS
 * uses is made here, once.  sb_set_table clears the release dates; setting or clearing them ends the current
 * search (sb_search_init again). */
int sb_set_release(sb_handle* h, const float* r, int J);
/* Per-job late penalties for SB_FLAG_LATE_PENALTY and SB_FLAG_COMPLETION_PENALTY: p host fp32 [J], the fixed cost
 * of each job that completes after its due date, every value finite and >= 0 with J * max_j p_j < 2^126 (else
 * SB_ERR_ARG, as is a J that differs from the table's); -0 is stored as +0.  p = NULL clears them.  SB_ERR_STATE
 * before sb_set_table.  sb_set_table clears the penalties; setting or clearing them ends the current search
 * (sb_search_init again).  Their sum is recorded for the search's temperature unit. */
int sb_set_penalty(sb_handle* h, const float* p, int J);
/* Runtime scenarios for SB_FLAG_WORST_MAKESPAN, SB_FLAG_MEAN_MAKESPAN, SB_FLAG_WORST_TARDINESS and
 * SB_FLAG_MEAN_TARDINESS: f fp32 [K][J], host or device, one positive
 * factor per scenario and job; scenario k's table is T_k[j][c] = fp32(f[k][j] * T[j][c]) for every cell of row j, of
 * the full and of the reduced table alike (+inf stays +inf).  K outside 1..8, a J that differs from the table's, or a
 * factor that is <= 0, NaN or inf is SB_ERR_ARG.  f = NULL clears them.  SB_ERR_STATE before sb_set_table.
 * sb_set_table clears the scenarios; setting or clearing them ends the current search (sb_search_init again). */
int sb_set_scenarios(sb_handle* h, const float* f, int K, int J);
/* copy the reduced table back (host pointers, either may be NULL): tmin fp32 [J][8], args u8 [J][8].
 * This is the table the reference solver is actually given: Task.strategies[g] after the profiler's
 * min over executors (PerformanceEvaluator.py:101-115), read at milp.py:77-81. */
int sb_get_reduced(sb_handle* h, float* tmin, uint8_t* args);

/* ---- the measured kernel: makespan of B candidates ----------------------------------------
 * opt, prio, makespan_out: device pointers.  prio element width is 1 byte if J <= 256 else 2.
 * best_key (device, nullable): a uint64 the kernel atomically MINs with
 * (float_bits(makespan) << 32) | (id_base + b), i.e. an arg-min over everything folded in. */
int sb_eval(sb_handle* h, const uint8_t* opt, const void* prio, int64_t B, int64_t row_stride,
            unsigned flags, float* makespan_out, uint64_t* best_key, uint32_t id_base);

/* which kernel the last sb_eval / sb_eval_host on this handle used:
 * 9 = job-indexed rows where the tile kernel runs short of shared memory (J >= 1024, or a table that does not
 *     fit beside the tiles; 32-byte aligned rows, sb_eval only): the opt rows are re-ordered into schedule order
 *     on the device (a scratch buffer of B * row_stride bytes owned by the handle, grow-only) and scored by the
 *     position-major kernel as under 5 / 8,
 * 8 = position-major kernel with the table in global memory, read through L1 / L2 (a one-node table beyond one
 *     SM's shared memory), 7 = the same with the table split over the shared memory of CTA pairs (test hook),
 * 6 = the alternate warp-shuffle kernel (SB_FLAG_ALT_WARPSCAN),
 * 5 = position-major kernel (SB_FLAG_OPT_BY_POSITION): both rows streamed, 32 bytes per lane per load,
 * 4 = as 3 but with the runtime table read from global memory (it does not fit in shared memory; what
 *     sb_eval_host, whose speed is PCIe's, still takes),
 * 3 = tile kernel, opt rows by TMA bulk copy + prio rows streamed with 256-bit loads (rows 32-byte
 *     aligned: the fast path), 2 = tile kernel with TMA bulk copies of both rows (16-byte aligned),
 * 1 = tile kernel with plain row loads (unaligned rows),
 * 0 = generic kernel (rows read from global memory; J too large for shared-memory tiles) */
int sb_last_eval_path(sb_handle* h);

/* check B candidates (device pointers): every prio row is a permutation of 0..J-1 and every opt
 * byte names an existing table cell.  sb_eval does not validate; out-of-range bytes are undefined
 * behaviour there.  bad_rows (host) receives the number of offending rows.  Synchronous. */
int sb_validate(sb_handle* h, const uint8_t* opt, const void* prio, int64_t B, int64_t row_stride,
                unsigned flags, int64_t* bad_rows);

/* same through HOST buffers: chunked H2D copies, kernel, D2H of the makespans, pipelined on
 * two internal streams; returns when makespan_out (host) is complete.  This is the call shape a CPU
 * caller of the reference has (everything in host memory, milp.py:23). */
int sb_eval_host(sb_handle* h, const uint8_t* opt, const void* prio, int64_t B, int64_t row_stride,
                 unsigned flags, float* makespan_out);

/* ---- full plan of B candidates (slot-exact; used for decode and for parity tests) ---------
 * Replaces reading the start / occupancy variables back from the solved MILP: sta[n][g][t] and
 * tga[t][n][g] of milp.py:330-334 (one shared Integer start per task, milp.py:139-149,233-256).
 * start_out fp32 [B][J] and slotmask_out u32 [B][J] are indexed by JOB; bit g (g < 8) of the mask =
 * GPU slot g of the job's node, bits 16.. = node index.  Device pointers; start_out / slotmask_out
 * may be NULL. */
int sb_eval_full(sb_handle* h, const uint8_t* opt, const void* prio, int64_t B, int64_t row_stride,
                 unsigned flags, float* makespan_out, float* start_out, uint32_t* slotmask_out);
/* Under SB_FLAG_WORST_MAKESPAN, SB_FLAG_MEAN_MAKESPAN, SB_FLAG_WORST_TARDINESS or SB_FLAG_MEAN_TARDINESS (else
 * SB_ERR_ARG): the slot-exact score of B candidates and every scenario's score, the makespan M_k or the total
 * tardiness S_k, makespans_out fp32 [B][K] (device pointers; score_out may be NULL). */
int sb_eval_scenarios(sb_handle* h, const uint8_t* opt, const void* prio, int64_t B, int64_t row_stride,
                      unsigned flags, float* score_out, float* makespans_out);

/* decode ONE candidate given in host memory into host arrays (all [J]; any may be NULL) — everything
 * milp.py:330-352 extracts per task (start, occupied GPUs, selected option, node):
 * start, GPU mask within the node, strategy index s (for SB_FLAG_REDUCED the arg-min strategy of
 * the cell), gpu count k, node index.  makespan (nullable) receives the candidate's makespan. */
int sb_decode(sb_handle* h, const uint8_t* opt, const void* prio, unsigned flags, float* start,
              uint32_t* slotmask, uint8_t* strategy, uint8_t* gpus, uint8_t* node, float* makespan);

/* ---- multi-GPU exchange over NVLink peer memory ----------------------------------------------
 * The path shards by candidate id; its only exchange is one MIN of the packed 64-bit key per round.
 * Each rank owns a mailbox in HBM that every peer maps with CUDA IPC; a rank publishes {key, round} in
 * its own mailbox (release at system scope; fused into the tail of the evaluation kernel with
 * SB_FLAG_POST_KEY) and a one-warp kernel on every rank loads all mailboxes over NVLink (acquire at
 * system scope) until they show the round, then folds the MIN.  One process per GPU:
 *   sb_xchg_create  -> 64-byte IPC handle; all-gather the handles (any transport);
 *   sb_xchg_connect (all handles, rank order);
 *   per round: sb_eval(..., flags | SB_FLAG_POST_KEY, ..., best_key, ...)  [or sb_xchg_post(key)]
 *              sb_xchg_reduce(out, fold)   — every rank must post and reduce every round;
 *   sb_xchg_check: synchronous; reports a timed-out wait (a peer never posted).
 * There is no reference counterpart (the reference solver is a single CPU process). */
int sb_xchg_create(sb_handle* h, int rank, int world, void* handle_out /* SB_IPC_HANDLE_BYTES */);
int sb_xchg_connect(sb_handle* h, const void* handles /* [world][SB_IPC_HANDLE_BYTES] */);
/* One process driving several devices (one handle per device, rank = position in `handles`): the mailboxes
 * are wired directly — same address space, cudaDeviceEnablePeerAccess, no IPC handles.  Replaces
 * sb_xchg_create + sb_xchg_connect for that case; the per-round calls are the same. */
int sb_xchg_connect_local(sb_handle** handles, int n);
int sb_xchg_post(sb_handle* h, const uint64_t* key_dev);
/* out_dev receives the MIN over all ranks; fold_dev (nullable) is MIN-ed with it in place */
int sb_xchg_reduce(sb_handle* h, uint64_t* out_dev, uint64_t* fold_dev);
int sb_xchg_check(sb_handle* h);

/* ---- search (replaces prob.solve(), milp.py:321-327) ---------------------------------------
 * A population of `chains` candidates lives on the device.  sb_search_init seeds it (random
 * valid options + random / LPT-like priorities, optionally chain 0 from a caller-supplied
 * warm-start candidate = the `presolved` plan of milp.py:35,103-104,151-155,197-202).
 * sb_search_round runs `rounds` Metropolis rounds: mutate -> evaluate (the sb_eval kernel) ->
 * accept, all on the device, and updates the best key.  The caller may exchange
 * best keys between GPUs (one MIN all-reduce of a uint64 per round) through
 * sb_search_best_key_ptr, and re-seed from a foreign elite with sb_search_inject. */
typedef struct sb_search_params {
  uint64_t seed;        /* RNG stream; candidate ids are global so ranks differ by chain_base */
  int64_t chains;       /* candidates in this GPU's population */
  uint64_t chain_base;  /* global id of chain 0 (rank * chains) */
  unsigned flags;       /* SB_FLAG_* */
  float t_start;        /* initial temperature as a fraction of the incumbent makespan (SB_FLAG_SUM_COMPLETION:
                         * of the incumbent's mean completion time, its sum / J; with SB_FLAG_WEIGHTED its
                         * weighted sum / the sum of the weights; with SB_FLAG_DUE the unit of SB_FLAG_DUE) */
  float t_end;          /* final temperature fraction */
  int total_rounds;     /* cooling horizon */
  int resample_every;   /* > 0: sb_search_round itself resamples the population by tournament before every round r
                         * with (r - 1) % resample_every == 0 — inside the round kernel where the rows are resident
                         * in shared memory (rivals = the 32 chains of a warp, re-dealt between launches), with the
                         * sb_search_resample kernel otherwise.  0: only when the caller calls sb_search_resample.  -1: automatic
                         * (2 where the tournament runs inside the round kernel, 4 where it is a copy of the population). */
} sb_search_params;

int sb_search_init(sb_handle* h, const sb_search_params* p, const uint8_t* warm_opt /*host, nullable*/,
                   const void* warm_prio /*host, nullable*/);
/* `rounds` Metropolis rounds, asynchronous on the handle's stream.  Fused rounds are issued up to 16 per launch:
 * a warp keeps its 32 chains' rows on chip and runs the rounds back to back (a rejected move is undone in
 * place, an accepted one writes its few changed bytes through to HBM); a chain whose candidate beats the incumbent
 * saved before the launch stops moving until the launch ends, so the saved incumbent is exactly the candidate
 * its key was scored on — and a search is reproducible bit for bit whatever the interleaving of warps. */
int sb_search_round(sb_handle* h, int rounds);
/* device pointer to the uint64 best key ((makespan bits << 32) | global chain id); after every call it is the key
 * sb_search_best returns with the saved candidate */
int sb_search_best_key_ptr(sb_handle* h, uint64_t** key_dev);
/* copy the best candidate found so far to host buffers: opt u8 [J], prio u8/u16 [J] */
int sb_search_best(sb_handle* h, uint8_t* opt, void* prio, float* makespan, uint64_t* key);
/* overwrite chains [first_chain, first_chain + copies) — the last `copies` chains if first_chain < 0 —
 * with the given candidate (host buffers), score them and fold them into the best key */
int sb_search_inject(sb_handle* h, const uint8_t* opt, const void* prio, int64_t first_chain, int copies);
/* tournament resampling: every chain continues from a random rival's candidate if the rival's
 * current makespan is strictly better (keeps the population concentrated on good basins) */
int sb_search_resample(sb_handle* h);
/* ---- the whole single-GPU search in one call (what prob.solve(solver) is to the reference, milp.py:321-327)
 * sb_search_seed_lpt plants three longest-processing-time candidates (every job on its fastest option / on its
 * least GPU-seconds option / in between; nodes filled greedily by GPU-seconds) into an eighth of the
 * population each and scores them; with SB_FLAG_SUM_COMPLETION the orders are shortest-processing-time
 * instead (ascending runtime of the chosen option), with SB_FLAG_WEIGHTED as well WSPT orders (ascending runtime / weight,
 * ties by job index), with SB_FLAG_DUE EDD orders (ascending due date, ties by runtime / weight, then job index),
 * same options and node fill.  Every job's option is one the search would propose: a cell below the sentinel, or
 * for a job without one its cheapest finite cell.  sb_search_run = sb_search_init + seeds + `rounds` rounds in groups of
 * `sync_every` (tournament resampling every `resample_every` rounds inside a group is only another launch;
 * the host reads the incumbent key once per group and applies the stopping rules) + sb_search_best.
 * The multi-GPU driver (saturn_b200/search.py) runs the same steps with a key exchange per group. */
typedef struct sb_search_control {
  int rounds;             /* >= 1 */
  int resample_every;     /* 0 = never, -1 = automatic; overrides sb_search_params.resample_every */
  int sync_every;         /* rounds per group, >= 1 */
  int patience;           /* stop after this many rounds without improvement; 0 = off */
  int heuristic_seeds;    /* 1 = sb_search_seed_lpt after initialisation */
  float target_makespan;  /* stop once the incumbent is <= this; <= 0 = off */
  double time_budget_s;   /* wall-clock budget (the reference's timeLimit); <= 0 = none */
  /* optional trace, one entry per group (NULL / 0 = none) */
  int history_cap;
  int* history_len;
  double* history_wall_s;
  int64_t* history_evaluated;
  float* history_makespan;
} sb_search_control;
typedef struct sb_search_result {
  float makespan;
  uint64_t key;        /* (float bits << 32) | global chain id of the incumbent */
  int64_t evaluated;   /* candidates scored */
  int rounds;          /* rounds run */
  int stop_reason;     /* 0 rounds exhausted, 1 time budget, 2 patience, 3 target reached (SB_FLAG_DUE: also a
                        * score of +0, which no plan can beat) */
  double wall_s;
} sb_search_result;
int sb_search_seed_lpt(sb_handle* h);
int sb_search_run(sb_handle* h, const sb_search_params* p, const sb_search_control* c, const uint8_t* warm_opt,
                  const void* warm_prio, uint8_t* opt_out /*host [J]*/, void* prio_out /*host [J]*/,
                  sb_search_result* result);
/* The same search sharded over the `n` devices of ONE process (one handle per device, the same table set on
 * each): the reference calls its solver from a single process (saturn/orchestrator.py:21-23,55,69), so this
 * is the call that lets that call site use every GPU of the node without torchrun.  Device i runs its own
 * population of p->chains chains with global ids p->chain_base + i * chains (counter-based RNG: the run is
 * identical to n single-device processes with those chain bases); after every group of `sync_every` rounds
 * the devices exchange one uint64 through the NVLink mailboxes (sb_xchg_connect_local is called if the
 * handles are not wired yet) and the host applies the stopping rules to the folded key.  The winner is read
 * from the device that owns its chain id.  result->evaluated counts all devices.  n = 1 is sb_search_run. */
int sb_search_run_multi(sb_handle** handles, int n, const sb_search_params* p, const sb_search_control* c,
                        const uint8_t* warm_opt, const void* warm_prio, uint8_t* opt_out /*host [J]*/,
                        void* prio_out /*host [J]*/, sb_search_result* result);
/* Population size that fills the device exactly once with the round kernel this table gets (resident warps
 * per SM x 32 lanes x SMs).  A population that is a whole multiple of it leaves no partially filled last
 * wave: 131,072 chains on 132 SMs x 12 warps are 2.6 waves and cost 3.  A combination of objective flags that sb_eval
 * refuses is SB_ERR_ARG here too. */
int sb_search_wave(sb_handle* h, unsigned flags, int64_t* chains);
/* 1 if rounds run as ONE fused kernel (move + evaluate + accept), 0 if they run as propose / evaluate /
 * accept kernels.  Fused rounds keep both rows of a tile's 32 candidates in shared memory when they fit
 * (all moves); for larger J the population is held in schedule order (opt by position) and both rows
 * stream through registers, with the move patched into the stream on the fly (no re-insertion moves).
 * That layout is internal: every function of this header takes and returns job-indexed opt rows.  All
 * forms are the same Metropolis search; move mixes and RNG streams differ slightly. */
int sb_search_is_fused(sb_handle* h);
/* sb_validate on the search population as it stands (every chain's rows: a permutation and existing table
 * cells), whatever encoding the population is kept in.  Synchronous; bad_rows (host) = offending chains. */
int sb_search_validate(sb_handle* h, int64_t* bad_rows);
/* Test hook.  Fused rounds of the tile kernel score a proposal incrementally: the chains of a warp make their
 * moves inside one window of 32 schedule positions per round and resume the list schedule from the state
 * snapshotted in front of that window.  With bit 0x08000000 set in sb_search_params.flags every such score is
 * also recomputed from position 0; this returns how many differed (must be 0).  Bits 0x10000000 (same
 * windowed moves, always scored from position 0) and 0x04000000 (round-1 move generator) select the
 * reference behaviours the tests and profiles compare against. */
int sb_search_verify_count(sb_handle* h, uint64_t* mismatches);
/* Test hooks of the streamed tile kernel (sb_eval path 3), kept on the handle for every later sb_eval until changed
 * (0 = none, the default).  Bit 1: every warp adds up the %globaltimer nanoseconds from issuing each tile's row
 * fetch to the fetch's completion, and its whole time in the tile loop, into two counters of the handle.  Bit 2:
 * one bulk copy per opt row even where the rows of a tile could be fetched with one.  Bit 4: every warp of a CTA
 * starts at once (no staggered phases).  None of them changes a result. */
int sb_debug_tile_options(sb_handle* h, unsigned options);
/* out[0] = the summed fetch waits, out[1] = the summed tile-loop times (ns) of every launch under option bit 1
 * since the last call; the call resets both.  Synchronous. */
int sb_debug_tile_wait(sb_handle* h, uint64_t* out);
/* Copy chains [first, first + count) of the search population to host buffers (any may be NULL): the current opt
 * rows u8 [count][J], job-indexed in this header's encoding whatever layout the population is kept in, the prio rows
 * u8/u16 [count][J] and the current scores fp32 [count] (the makespan, or the objective's score).  *layout receives
 * how rounds run on it: 0 = propose / evaluate / accept kernels, 1 = the fused tile round, 2 = the position-major
 * round.  For tests that check the state every chain is left in.  Synchronous. */
int sb_debug_search_population(sb_handle* h, int64_t first, int64_t count, uint8_t* opt, void* prio, float* score,
                               int* layout);
/* candidates evaluated so far by this handle's searches */
int sb_search_stats(sb_handle* h, int64_t* evaluated, int64_t* rounds_done);

#ifdef __cplusplus
}
#endif
#endif /* SATURN_B200_H */
