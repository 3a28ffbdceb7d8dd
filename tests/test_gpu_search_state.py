"""The state every chain of the search population is left in, checked after every step of a scripted search.

The other search tests look at the incumbent only.  Here `Engine.debug_search_population` reads back every chain's
current rows and score (opt rows job-indexed whatever layout the population is kept in), and after each step (init
with and without a warm start, the heuristic seeds, rounds of 1, 3, 16 and 17 (two launches), a tournament
resample, and injections that clamp their range) the whole population is held to these invariants, exactly (float
bits and bytes):

  I1 score   every chain's score equals the fp32 C oracle's score of its rows (objective, release dates, nodes);
  I2 rows    every prio row is a permutation, every opt byte is one the search proposes (the rule of k_build_valid,
             recomputed here from the reduced table and the sentinel), nodes are below `nodes`;
  I3 key     the oracle score of search_best()'s rows is its key, the key's id is one of this population's chain
             ids, its score is <= every current score (every current candidate has been folded), and the
             population's best key (search_best_key) is that saved key;
  I4 tail    after a call of one launch without resampling that lowered the saved key, the winning chain holds
             exactly search_best()'s rows and its score equals the key;
  I5 greedy  at temperature 0 no chain's score increases across rounds and resamples (tournaments included);
  I6 copy    after search_resample every chain holds its own previous (rows, score) or another chain's previous
             pair with a strictly smaller score;
  I7 inject  injected ranges hold the candidate, every other chain is unchanged; with a warm start chain 0 is the
             warm candidate; after the heuristic seeds the seeded ranges equal lpt_seeds() (the last writer wins);
  I8 repro   the same parameters twice give the identical whole population after every step;
  I9 count   search_stats() evaluated = chains * (1 + rounds) + the injected copies.

The cases cover the three layouts (fused tile rounds, incremental or not; the propose / evaluate / accept kernels;
the position-major kernel), 1 to 8 nodes, the full table, all ten objectives with release dates off and on,
populations of 1 to one wave + 17 chains, random tables with masks and sentinel cells and tie-heavy tables (all
runtimes equal, or in {1, 2, 3}), where `<=` acceptance and `<` tournaments differ.
"""
import numpy as np
import pytest

from oracle import ref_eval as R
from oracle import ref_exact as X
from oracle import ref_release as RR
from saturn_b200 import _lib
from saturn_b200.engine import OBJECTIVES
from saturn_b200.search import lpt_seeds

SENTINEL = 1.0e6
CHAIN_BASE = 1000
TOTAL_ROUNDS = 40
LAYOUTS_SEEN = set()


# --------------------------------------------------------------------------- tables and per-job data
def make_table(family, J, S, seed):
    """T[J][S][8] fp32, gcount = 1..8.  "rnd": synth_table (masked strategies, 1e8 failures at k <= 2) plus 1e6
    "not profiled" and +inf cells, and two jobs with no cell below the sentinel; "small": runtimes in {1, 2, 3};
    "equal": every runtime 2.5; "seedtrap": "small" with jobs 0 and 1 as in the seed-fallback example (job 0: 1e6 on
    k = 1, 5e5 on k = 8; job 1: 1e8 on k = 1, 1e6 on k = 4; every other cell of both +inf)."""
    rng = np.random.default_rng(seed)
    if family == "rnd":
        T, _ = R.synth_table(J, S, 8, seed=seed)
        pick = rng.uniform(size=T.shape)
        T[(pick < 0.04) & (T < SENTINEL)] = SENTINEL
        T[pick > 0.97] = np.inf
        for j in rng.choice(J, size=min(2, J), replace=False):
            T[j] = 1e8
            T[j, rng.integers(0, S), rng.integers(0, 8)] = SENTINEL
        for j in range(J):                              # keep a finite cell in every job
            if not np.isfinite(T[j]).any():
                T[j, 0, 0] = 1e8
    elif family in ("small", "seedtrap"):
        T = rng.integers(1, 4, (J, S, 8)).astype(np.float32)
        if family == "seedtrap":
            T[:2] = np.inf
            T[0, :, 0], T[0, :, 7] = 1e6, 5e5
            T[1, :, 0], T[1, :, 3] = 1e8, 1e6
    elif family == "equal":
        T = np.full((J, S, 8), 2.5, dtype=np.float32)
    else:
        raise ValueError(family)
    return T.astype(np.float32)


def proposable(tmin, args, reduced, sentinel=SENTINEL):
    """ok[J][256]: the opt bytes (option bits only, without the node) the search proposes for each job, by the rule of
    k_build_valid: every column below the sentinel, coded (args << 3) | col on the full table; a job with none keeps
    its first cheapest finite column (column 0 if it has no finite cell)."""
    J = tmin.shape[0]
    col = np.arange(8)[None, :]
    code = np.broadcast_to(col, (J, 8)) if reduced else (args.astype(np.int64) << 3) | col
    use = tmin < sentinel
    bare = ~use.any(axis=1)
    first_min = np.where(np.isfinite(tmin).any(axis=1), np.argmin(tmin, axis=1), 0)
    use[bare, first_min[bare]] = True
    ok = np.zeros((J, 256), dtype=bool)
    rows, cols = np.nonzero(use)
    ok[rows, code[rows, cols]] = True
    return ok


def per_job(T, objective, release, ints, seed):
    """fp32 weights / due dates / release dates at the scale of the table's plans, as the objective's flag bits need
    them."""
    rng = np.random.default_rng(seed)
    J = T.shape[0]
    usable = np.where(T < SENTINEL, T, np.inf).min(axis=(1, 2))
    usable = np.where(np.isfinite(usable), usable, 1.0)
    horizon = float(usable.sum()) / 4 + 1.0
    integral = bool((T[np.isfinite(T)] == np.round(T[np.isfinite(T)])).all())
    w = d = r = None
    use_w, use_d = X.needs(objective)
    if use_w:
        w = rng.choice([0.5, 1.0, 2.0, 3.0], J).astype(np.float32)
    if use_d:
        d = rng.uniform(-0.05, 1.0, J) * horizon
        d = (np.round(d) if integral else d).astype(np.float32)
    if release:
        r = rng.uniform(-0.1, 0.5, J) * horizon
        r = (np.round(r) if integral else r).astype(np.float32)
    return w, d, r


# --------------------------------------------------------------------------- the oracle
class Ctx:
    def __init__(self, engine, case, T):
        self.J = T.shape[0]
        self.nodes, self.reduced, self.ints, self.objective = case["nodes"], case["reduced"], case["ints"], case["objective"]
        self.tmin, self.args = engine.reduced_table()
        self.tab = self.tmin[:, None, :] if self.reduced else R.canon_table(T, range(1, 9))
        self.ok = proposable(self.tmin, self.args, self.reduced)
        self.w, self.d, self.r = engine.weights, engine.due, engine.release
        self.pdt = np.uint8 if self.J <= 256 else np.uint16

    def score(self, opt, prio):
        """fp32 scores of rows opt[B][J], prio[B][J] (the C ports, bit-exact with the kernels)."""
        r = np.zeros(self.J, np.float32) if self.r is None else self.r
        return RR.c_evaluate(self.tab, np.ascontiguousarray(opt), np.ascontiguousarray(prio), r, self.ints, np.float32,
                             nodes=self.nodes, objective=self.objective, weights=self.w, due=self.d)

    def candidate(self, rng):
        """A random candidate built from proposable cells only (job-indexed opt row, prio row)."""
        opt = np.empty(self.J, dtype=np.uint8)
        for j in range(self.J):
            opt[j] = rng.choice(np.nonzero(self.ok[j])[0])
        if self.nodes > 1:
            opt |= (rng.integers(0, self.nodes, self.J) << 3).astype(np.uint8)
        return opt, rng.permutation(self.J).astype(self.pdt)

    def seeds(self):
        """The heuristic seeds as sb_search_seed_lpt plants them (job-indexed opt rows in the search's encoding)."""
        out = []
        for col, order in lpt_seeds(self.tmin, sentinel=SENTINEL, nodes=self.nodes, objective=self.objective,
                                    weights=self.w, due=self.d, release=self.r, integer_starts=self.ints):
            opt = col if self.reduced else (self.args[np.arange(self.J), col & 7] << 3) | col
            out.append((opt.astype(np.uint8), order.astype(self.pdt)))
        return out


def bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def check_state(engine, ctx, chains, label):
    """I1, I2 and I3 on the whole population; returns it as (opt, prio, score, layout)."""
    opt, prio, score, layout = engine.debug_search_population()
    J = ctx.J
    assert opt.shape == (chains, J) and layout in (0, 1, 2), label
    # I2: permutations, proposable options, nodes
    srt = np.sort(prio.astype(np.int64), axis=1)
    bad = np.nonzero((srt != np.arange(J)).any(axis=1))[0]
    assert len(bad) == 0, (label, "prio row not a permutation", bad[:5])
    byte = opt & 7 if ctx.nodes > 1 else opt
    if ctx.nodes > 1:
        assert ((opt >> 3) < ctx.nodes).all(), (label, "node out of range")
    okb = ctx.ok[np.arange(J)[None, :], byte]
    if not okb.all():
        c, j = np.argwhere(~okb)[0]
        raise AssertionError((label, "opt byte not proposable", int(c), int(j), int(opt[c, j]), ctx.tmin[j].tolist()))
    # I1: every chain's score
    ref = ctx.score(opt, prio)
    diff = np.nonzero(bits(ref) != bits(score))[0]
    assert len(diff) == 0, (label, "score != oracle", diff[:5], score[diff[:5]], ref[diff[:5]])
    # I3: the saved incumbent
    bo, bp, bmk, key = engine.search_best()
    kbits = key >> 32
    assert int(bits(ctx.score(bo[None], bp[None]))[0]) == kbits, (label, "incumbent's rows do not score its key")
    assert int(bits(np.float32(bmk))[0]) == kbits, label
    assert CHAIN_BASE <= (key & 0xffffffff) < CHAIN_BASE + chains, (label, "key id outside the population")
    # the population's best key names the saved incumbent: a lower key left behind would make the next save copy the
    # rows its chain holds by then
    assert int(engine.search_best_key().item()) == key, (label, "best key != saved key", hex(key))
    assert np.float32(bmk) <= score.min(), (label, "a current score beats the saved key", bmk, score.min())
    return opt, prio, score, layout


def expect_inject(pop, chains, cand, first, copies):
    """The population after sb_search_inject(cand, first, copies), the range clamped as the library clamps it."""
    copies = min(copies, chains)
    f = chains - copies if first < 0 else first
    if f + copies > chains:
        f = chains - copies
    opt, prio = pop[0].copy(), pop[1].copy()
    opt[f:f + copies] = cand[0]
    prio[f:f + copies] = cand[1]
    return opt, prio, f, copies


def assert_rows(pop, opt, prio, label, keep_scores=None):
    diff = np.nonzero((pop[0] != opt).any(axis=1) | (pop[1] != prio).any(axis=1))[0]
    assert len(diff) == 0, (label, "rows differ from the expected population", diff[:5])
    if keep_scores is not None:
        sel, old = keep_scores
        assert np.array_equal(bits(pop[2][sel]), bits(old)), (label, "an untouched chain's score changed")


# --------------------------------------------------------------------------- the scripted search
def run_script(engine, case):
    """Set up the case, run the scripted search and check every invariant after every step.  Returns the digest of
    every step's whole population (I8) and the layouts seen."""
    seed = case["seed"]
    rng = np.random.default_rng(seed)
    T = make_table(case["family"], case["J"], case["S"], seed)
    engine.set_table(T, nodes=case["nodes"], sentinel=SENTINEL)
    w, d, r = per_job(T, case["objective"], case["release"], case["ints"], seed + 1)
    if w is not None:
        engine.set_weights(w)
    if d is not None:
        engine.set_due(d)
    if r is not None:
        engine.set_release(r)
    ctx = Ctx(engine, case, T)
    chains = case["chains"]
    if chains == "wave+17":
        chains = engine.search_wave(reduced=case["reduced"]) + 17
    t = 0.0 if case["t0"] else 0.02
    warm = ctx.candidate(rng) if case["warm"] else None
    resample = case["resample"]
    engine.search_init(chains, seed=seed, chain_base=CHAIN_BASE, integer_starts=case["ints"], reduced=case["reduced"],
                       t_start=t, t_end=t * 0.005, total_rounds=TOTAL_ROUNDS, warm=warm, resample_every=resample,
                       _no_fused=case["no_fused"], _extra_flags=case["hooks"], objective=case["objective"])
    label = (case["name"], "init")
    injected = 0
    pop = check_state(engine, ctx, chains, label)
    if warm is not None:
        assert np.array_equal(pop[0][0], warm[0]) and np.array_equal(pop[1][0], warm[1]), (label, "warm start")
    digests = [(pop[0].tobytes(), pop[1].tobytes(), pop[2].tobytes())]
    layouts = {pop[3]}

    def counters(label):
        ev, rounds = engine.search_stats()
        assert ev == chains * (1 + rounds) + injected, (label, ev, rounds, injected)

    counters(label)
    # the heuristic seeds: an eighth of the population each, the last writer wins
    per = max(1, chains // 8)
    exp_o, exp_p = pop[0].copy(), pop[1].copy()
    for i, (so, sp) in enumerate(ctx.seeds()):
        first = min(i * per, max(0, chains - per))
        exp_o, exp_p, _, n = expect_inject((exp_o, exp_p), chains, (so, sp), first, min(per, chains))
        injected += n
    engine.search_seed_lpt()
    label = (case["name"], "seed")
    new = check_state(engine, ctx, chains, label)
    assert_rows(new, exp_o, exp_p, label)
    untouched = np.ones(chains, dtype=bool)
    untouched[:min(chains, 2 * per + per)] = False
    untouched[max(0, chains - per):] = False
    assert np.array_equal(bits(new[2][untouched]), bits(pop[2][untouched])), label
    counters(label)
    pop = new
    digests.append((pop[0].tobytes(), pop[1].tobytes(), pop[2].tobytes()))

    steps = [("round", 1), ("round", 3), ("resample",), ("round", 16), ("round", 17), ("resample",),
             ("inject", -1, 3), ("inject", chains - 2, 5), ("round", 3), ("inject", 0, chains + 7), ("round", 1)]
    for step in steps:
        label = (case["name"],) + step
        old = pop
        if step[0] == "round":
            n = step[1]
            key_before = engine.search_best()[3]
            engine.search_round(n)
            pop = check_state(engine, ctx, chains, label)
            # I4: one launch, no resampling, a lower saved key -> the winning chain holds the saved rows
            one_launch = n == 1 or (pop[3] in (1, 2) and n <= 16)
            bo, bp, bmk, key = engine.search_best()
            if one_launch and resample == 0 and key < key_before:
                c = (key & 0xffffffff) - CHAIN_BASE
                assert np.array_equal(pop[0][c], bo) and np.array_equal(pop[1][c], bp), (label, "I4 rows", c)
                assert int(bits(pop[2][c:c + 1])[0]) == key >> 32, (label, "I4 score", c)
        elif step[0] == "resample":
            engine.search_resample()
            pop = check_state(engine, ctx, chains, label)
            # I6: own pair, or another chain's previous pair with a strictly smaller score
            prev = {}
            for c in range(chains):
                prev.setdefault(old[0][c].tobytes() + old[1][c].tobytes(), set()).add(int(bits(old[2][c:c + 1])[0]))
            same = (pop[0] == old[0]).all(axis=1) & (pop[1] == old[1]).all(axis=1) & (bits(pop[2]) == bits(old[2]))
            for c in np.nonzero(~same)[0]:
                sb = int(bits(pop[2][c:c + 1])[0])
                assert pop[2][c] < old[2][c], (label, "I6: took a rival that is not strictly better", c)
                assert sb in prev.get(pop[0][c].tobytes() + pop[1][c].tobytes(), ()), (label, "I6: not a copy", c)
        else:
            _, first, copies = step
            cand = ctx.candidate(rng)
            exp_o, exp_p, f, n = expect_inject(old, chains, cand, first, copies)
            engine.search_inject(cand[0], cand[1], copies=copies, first=first)
            injected += n
            pop = check_state(engine, ctx, chains, label)
            keep = np.ones(chains, dtype=bool)
            keep[f:f + n] = False
            assert_rows(pop, exp_o, exp_p, label, keep_scores=(keep, old[2][keep]))
        if case["t0"] and step[0] in ("round", "resample"):
            up = np.nonzero(pop[2] > old[2])[0]
            assert len(up) == 0, (label, "I5: a score rose at temperature 0", up[:5], old[2][up[:5]], pop[2][up[:5]])
        counters(label)
        layouts.add(pop[3])
        digests.append((pop[0].tobytes(), pop[1].tobytes(), pop[2].tobytes()))
    return digests, layouts


def case(name, J, chains, layout=None, S=1, nodes=1, reduced=True, objective="makespan", release=False,
         family="rnd", ints=True, hooks=0, no_fused=False, resample=0, t0=False, warm=False, twice=False):
    return dict(name=name, J=J, S=S, nodes=nodes, reduced=reduced, chains=chains, objective=objective, release=release,
                family=family, ints=ints, hooks=hooks, no_fused=no_fused, resample=resample, t0=t0, warm=warm,
                twice=twice, layout=layout, seed=len(CASES) * 7919 + J)


NOINC, ROUND1 = _lib.HOOK_NO_INCREMENTAL, _lib.HOOK_ROUND1_MOVES
CASES = []
for _c in [
    # fused tile rounds (layout 1, u8 priorities: from J = 257 on, u16 rows for 8 warps no longer fit in shared
    # memory and the population is position-major), incremental unless hooked off
    ("tile_J40", 40, 33, 1, dict(S=2, warm=True, twice=True)),
    ("tile_J100_tie_t0", 100, 1000, 1, dict(family="small", resample=-1, t0=True)),
    ("tile_J256", 256, 4097, 1, dict(ints=False, warm=True)),
    ("tile_J256_equal_t0", 256, 1000, 1, dict(family="equal", resample=-1, t0=True, twice=True)),
    ("tile_J40_one", 40, 1, 1, dict(resample=-1)),
    ("tile_J40_31", 40, 31, 1, dict(family="small", resample=-1, t0=True)),
    ("tile_J40_wave", 40, "wave+17", 1, dict(resample=-1, warm=True)),
    ("noinc_J100", 100, 31, 1, dict(hooks=NOINC, family="small")),
    ("noinc_J256_t0", 256, 1000, 1, dict(hooks=NOINC, resample=-1, t0=True)),
    ("noinc_J40_tie", 40, 4097, 1, dict(hooks=NOINC, family="small", resample=-1)),
    ("round1_J256", 256, 33, 1, dict(hooks=ROUND1, warm=True)),
    ("round1_J100_t0", 100, 1000, 1, dict(hooks=ROUND1, family="small", resample=-1, t0=True)),
    ("round1_J200_equal", 200, 4097, 1, dict(hooks=ROUND1, family="equal", resample=-1)),
    # J = 300: u16 priorities, position-major, with the same hooks
    ("pos_J300_equal_t0", 300, 1000, 2, dict(family="equal", resample=-1, t0=True)),
    ("pos_J300", 300, 31, 2, dict(resample=2)),
    ("pos_noinc_J300", 300, 1000, 2, dict(hooks=NOINC, resample=-1, t0=True)),
    ("pos_round1_J300_tie", 300, 4097, 2, dict(hooks=ROUND1, family="small", resample=-1)),
    # propose / evaluate / accept kernels and the copy tournament (layout 0)
    ("unfused_J100", 100, 1000, 0, dict(no_fused=True, warm=True, twice=True)),
    ("unfused_J256_tie_t0", 256, 33, 0, dict(no_fused=True, family="small", resample=-1, t0=True)),
    ("unfused_J40_one", 40, 1, 0, dict(no_fused=True, resample=-1)),
    ("unfused_J300_equal", 300, 4097, 0, dict(no_fused=True, family="equal", resample=-1)),
    # several nodes, fused
    ("nodes2_J100", 100, 1000, None, dict(nodes=2, warm=True)),
    ("nodes3_J64_tie_t0", 64, 31, None, dict(nodes=3, family="small", resample=-1, t0=True)),
    ("nodes8_J200", 200, 4097, None, dict(nodes=8, resample=-1)),
    # position-major populations (layout 2)
    ("pos_J700", 700, 1000, 2, dict(warm=True, twice=True)),
    ("pos_J1024_tie_t0", 1024, 33, 2, dict(family="small", resample=-1, t0=True)),
    ("pos_J2100", 2100, 300, 2, dict(resample=-1)),
    ("pos_J700_nodes2", 700, 1000, 2, dict(nodes=2, warm=True)),
    ("pos_J1024_equal", 1024, 31, 2, dict(family="equal", resample=-1, t0=True)),
    # the full table (strategy bits in the opt bytes)
    ("full_S3_J64", 64, 1000, None, dict(S=3, reduced=False, warm=True)),
    ("full_S8_J64_t0", 64, 33, None, dict(S=8, reduced=False, family="small", resample=-1, t0=True)),
    ("full_S3_J256_tie", 256, 4097, None, dict(S=3, reduced=False, family="small", resample=-1)),
    ("full_S8_J256", 256, 1000, None, dict(S=8, reduced=False, ints=False)),
    # the seed-fallback example embedded in a J = 64 table
    ("seedtrap_reduced", 64, 33, None, dict(family="seedtrap")),
    ("seedtrap_full", 64, 1000, None, dict(family="seedtrap", S=2, reduced=False)),
    ("seedtrap_nodes2", 64, 31, None, dict(family="seedtrap", nodes=2, resample=-1)),
    # forms whose scores tie in bulk: a late count on equal runtimes at temperature 0, a max fold on the full table and
    # on 8 nodes
    ("late_tasks_equal_t0", 256, 1000, 1, dict(objective="late_tasks", family="equal", resample=-1, t0=True)),
    ("wmax_tardiness_full_S3", 64, 1000, None, dict(S=3, reduced=False, objective="weighted_max_tardiness",
                                                     release=True, warm=True)),
    ("max_lateness_nodes8", 200, 4097, None, dict(nodes=8, objective="max_lateness", resample=-1)),
]:
    CASES.append(case(_c[0], _c[1], _c[2], _c[3], **_c[4]))

# every objective, release dates off and on, at J in {256, 700} on 1 and 2 nodes
_SHAPES = [(256, 1), (700, 1), (256, 2), (700, 2)]
for _i, _obj in enumerate(OBJECTIVES):
    for _k, _rel in enumerate((False, True)):
        _J, _n = _SHAPES[(2 * _i + _k) % 4]
        CASES.append(case("%s_%s_J%d_n%d" % (_obj, "rel" if _rel else "norel", _J, _n), _J, 1000 if _J == 256 else 300,
                          None, nodes=_n, objective=_obj, release=_rel, family="small" if _k else "rnd",
                          resample=-1 if _i % 2 else 0, t0=_i % 5 == 4, warm=_k == 1, twice=_i % 5 == 3 and _k == 1))


# --------------------------------------------------------------------------- CPU
def test_seeds_use_only_proposable_cells():
    """On random masked tables with sentinel-only jobs, under every objective and 1..3 nodes, every seed's option is
    one the search proposes (the set recomputed here by the rule of k_build_valid)."""
    for seed in range(6):
        T = make_table("rnd" if seed % 2 == 0 else "seedtrap", 64, 3, seed)
        tab = R.canon_table(T, range(1, 9))
        tmin, args = R.reduce_table(tab)
        ok = proposable(tmin, args, reduced=True)
        w, d, r = per_job(T, RR.OBJECTIVES[seed % 5], seed % 2 == 1, True, seed)
        for nodes in (1, 2, 3):
            for col, order in lpt_seeds(tmin, sentinel=SENTINEL, nodes=nodes, objective=RR.OBJECTIVES[seed % 5],
                                        weights=w, due=d, release=r):
                assert ok[np.arange(64), col & 7].all(), (seed, nodes)
                assert sorted(order.tolist()) == list(range(64))
                assert ((col >> 3) < nodes).all()


def test_proposable_set_matches_the_seed_fallback_example():
    """The rule the GPU tests hold the population to, on the example table: job 0 may use k = 8 only, job 1 only its
    cheapest cell k = 4 (no cell below the sentinel)."""
    T = make_table("seedtrap", 4, 1, 0)
    tmin, args = R.reduce_table(R.canon_table(T, range(1, 9)))
    ok = proposable(tmin, args, reduced=True)
    assert np.nonzero(ok[0])[0].tolist() == [7]
    assert np.nonzero(ok[1])[0].tolist() == [3]


# --------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_population_invariants(engine, c):
    digests, layouts = run_script(engine, c)
    if c["layout"] is not None:
        assert layouts == {c["layout"]}, (c["name"], layouts)
    LAYOUTS_SEEN.update(layouts)
    if c["twice"]:
        again, _ = run_script(engine, c)
        for i, (a, b) in enumerate(zip(digests, again)):
            assert a == b, (c["name"], "I8: the population differs between two identical runs at step", i)


@pytest.mark.gpu
def test_zz_every_population_layout_was_checked():
    """Runs after the cases: the fused tile rounds, the propose / evaluate / accept kernels and the position-major
    kernel each had their whole population checked."""
    if len(LAYOUTS_SEEN) == 0:
        pytest.skip("no population case ran")
    assert LAYOUTS_SEEN == {0, 1, 2}, LAYOUTS_SEEN
