"""GPU: the search + plan emission through the reference-facing API (saturn.solver.solve)."""
import numpy as np
import pytest
import torch

from conftest import tasks_from_tuples
from oracle import ref_eval as R

pytestmark = pytest.mark.gpu


def _check_plan(tasks, out):
    sta, tga, bss, bna, boa, mk = out
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, mk) == []
    plan = R.plan_from_arrays(tuples, sta, tga, bss, bna)
    ok, ov, mk2 = R.check_plan([p[0] for p in plan], [p[1] for p in plan], [p[2] for p in plan], [p[3] for p in plan])
    assert ok and ov == 0
    assert mk2 == pytest.approx(mk, rel=1e-12)
    return mk


def test_solve_matches_reference_milp_optimum(golden):
    """On every instance the reference MILP proved optimal, the GPU search returns a plan that is
    feasible under the reference's own constraints with makespan <= the MILP's (they coincide)."""
    import saturn.solver as ss
    n = 0
    for rec in golden["cases"]:
        if rec["variant"] != "tight_m" or not rec["incumbent"]:
            continue
        tasks = tasks_from_tuples(rec["gpu_time_tuples"])
        out = ss.solve(tasks, None, gurobi=False, threads=1, interval=1000, timeout=60, chains=8192, rounds=60)
        mk = _check_plan(tasks, out)
        assert mk <= rec["makespan"] * (1 + 1e-9), rec["name"]
        if rec["proven_optimal"]:
            assert mk == pytest.approx(rec["makespan"], rel=1e-9), rec["name"]
        npt, tdd, st = ss.convert_into_comprehensible(tasks, out[2], out[4], out[1], out[3], out[0])
        assert all(t.selected_strategy is not None for t in tasks)
        assert max(s + t.selected_strategy.runtime for s, t in zip(st, tasks)) == pytest.approx(mk, rel=1e-12)
        n += 1
    assert n >= 5


def test_solve_orchestrator_call_shapes():
    """orchestrator.py:55 binds (task_list, None, interval, interval//2, cpu_count) positionally, i.e.
    gurobi=1000, interval=500, timeout=cpu_count; :69 passes the previous tuple back as presolved."""
    from saturn_b200 import solve
    from saturn_b200 import solver as S
    rng = np.random.default_rng(5)
    tuples = [[(g, float(rng.uniform(300, 3000)) / g ** 0.7) for g in (1, 2, 4, 8)] for _ in range(12)]
    tasks = tasks_from_tuples(tuples)
    first = solve(tasks, None, gurobi=1000, threads=4, interval=500, timeout=8, chains=8192, rounds=40)
    mk1 = _check_plan(tasks, first)
    assert isinstance(first[5], float) and S.last_stats["adopted"]
    # second solve, default policy = the reference's observable behaviour: always adopt the fresh plan
    again = solve(tasks, first, True, 4, 100, 50, chains=8192, rounds=40)
    assert S.last_stats["adopted"] and again[5] <= mk1 * (1 + 1e-9)
    _check_plan(tasks, again)
    # opt-in hysteresis (documented intent): plan barely better -> keep the old plan shifted by `interval`
    second = solve(tasks, first, True, 4, 100, 50, chains=8192, rounds=40, hysteresis=True)
    assert not S.last_stats["adopted"]
    assert second[5] == pytest.approx(mk1 - 100)
    assert max(v for n in second[0] for g in n for v in g) == pytest.approx(max(max(v for n in first[0] for g in n for v in g) - 100, 0))
    # fewer tasks than the previous plan -> adopt the fresh plan (milp.py:394-399)
    third = solve(tasks[:7], first, True, 4, 100, 50, chains=8192, rounds=40)
    assert S.last_stats["adopted"] and len(third[1]) == 7
    _check_plan(tasks[:7], third)


def test_sentinel_options_never_selected():
    from saturn_b200 import Strategy, solve
    from conftest import DuckTask
    tasks = []
    rng = np.random.default_rng(1)
    for t in range(10):
        base = float(rng.uniform(500, 2000))
        strat = {}
        for g in range(1, 9):
            if g in (2, 4):
                strat[g] = Strategy("fsdp", g, {}, base / g ** 0.8)
            else:
                strat[g] = Strategy(None, g, None, 1000000)       # PerformanceEvaluator.py:99 initialisation
        tasks.append(DuckTask("t%d" % t, strat))
    out = solve(tasks, None, chains=4096, rounds=30)
    _check_plan(tasks, out)
    for row, t in zip(out[2], tasks):
        g = list(t.strategies.keys())[int(np.argmax(row))]
        assert g in (2, 4)


def test_search_quality_and_reproducibility(engine):
    """C3-shaped instance: the search beats the best of its own random initial population, the
    result decodes to a feasible plan, and a fixed seed reproduces the same incumbent."""
    from saturn_b200.search import run_search
    J, S, G = 64, 6, 8
    T, valid = R.synth_table(J, S, G, seed=0)
    engine.set_table(T)
    r1 = run_search(engine, chains=16384, rounds=60, seed=7, record_history=True, use_dist=False)
    r2 = run_search(engine, chains=16384, rounds=60, seed=7, use_dist=False)
    assert r1.makespan == r2.makespan and np.array_equal(r1.opt, r2.opt) and np.array_equal(r1.prio, r2.prio)
    assert r1.history[-1][2] < r1.history[0][2]
    assert r1.evaluated >= 16384 * 61
    tab = R.canon_table(T, range(1, 9))
    mk, start, mask, _ = R.list_schedule(tab, r1.opt, r1.prio, True, np.float32)
    assert mk == r1.makespan
    dec = engine.decode(r1.opt, r1.prio)
    assert dec["makespan"] == r1.makespan and list(dec["slotmask"]) == mask
    rt = tab[np.arange(J), r1.opt >> 3, r1.opt & 7]
    ok, ov, _ = R.check_plan(list(dec["start"]), list(dec["slotmask"]), list(rt), list(dec["gpus"]))
    assert ok
    assert (rt < 1e6).all()           # never proposes the 1e8 sentinel cells


def test_orchestrate_simulated_run():
    from saturn_b200 import orchestrate
    rng = np.random.default_rng(9)
    tuples = [[(g, float(rng.uniform(800, 5000)) / g ** 0.8) for g in (1, 2, 4, 8)] for _ in range(8)]
    tasks = tasks_from_tuples(tuples)
    for t in tasks:
        t.total_batches = 200
    launched = []
    recs = orchestrate(tasks, interval=1000, execute_fn=lambda rtt, btr, itv, npt, tdd: launched.append(len(rtt)),
                       solver_kwargs={"chains": 4096, "rounds": 25}, max_intervals=50)
    assert all(t.total_batches == 0 for t in tasks)
    assert len(recs) >= 2 and sum(launched) >= 8


def test_multi_node_solve_matches_reference_milp(golden_n2):
    """solve(nodes=2) on the instances the reference MILP solved with ray.nodes() == 2 nodes."""
    import saturn.solver as ss
    for rec in golden_n2["cases"]:
        tasks = tasks_from_tuples(rec["gpu_time_tuples"])
        out = ss.solve(tasks, None, gurobi=False, timeout=60, chains=8192, rounds=60, nodes=2)
        sta, tga, bss, bna, boa, mk = out
        assert len(sta) == 2 and len(bna[0]) == 2
        tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
        assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, mk) == []
        assert mk == pytest.approx(rec["makespan"], rel=1e-9), rec["name"]
        npt, tdd, st = ss.convert_into_comprehensible(tasks, bss, boa, tga, bna, sta)
        assert set(int(npt[t]) for t in tasks) == {0, 1}
        # warm start from the previous plan keeps working with nodes
        again = ss.solve(tasks, out, gurobi=False, timeout=60, chains=4096, rounds=20, nodes=2)
        assert again[5] <= mk * (1 + 1e-9)


@pytest.mark.parametrize("J,S,nodes", [(64, 6, 1), (256, 8, 1), (100, 1, 2), (400, 1, 1), (1024, 1, 1), (700, 1, 2)])
def test_fused_and_unfused_search_rounds(engine, J, S, nodes):
    """The fused round (move + evaluate + accept in one kernel) and the propose / evaluate / accept
    round are the same search: both improve on the seeded population, both return candidates whose
    oracle makespan equals the reported one, and the chain state they leave behind is consistent
    (re-evaluating the incumbent reproduces its key)."""
    from saturn_b200.search import run_search
    T, valid = R.synth_table(J, S, 8, seed=2, masked=(S > 1))
    engine.set_table(T, nodes=nodes)
    tab = R.canon_table(T, range(1, 9))
    reduced = nodes > 1 or J > 400
    if reduced:
        tab = R.reduce_table(tab)[0][:, None, :]
    res = {}
    for fused in (True, False):
        r = run_search(engine, chains=8192 if J <= 400 else 2048, rounds=40, seed=3, reduced=reduced or J > 400,
                       record_history=True, use_dist=False, _no_fused=not fused)
        assert engine.search_is_fused() == fused
        assert r.history[-1][2] < r.history[0][2]
        mk = R.list_schedule(tab, r.opt, r.prio, True, np.float32, nodes=nodes)[0]
        assert mk == r.makespan
        assert sorted(r.prio.tolist()) == list(range(J))
        res[fused] = r.makespan
    assert abs(res[True] / res[False] - 1) < (0.02 if J <= 400 else 0.05)


@pytest.mark.parametrize("J,nodes", [(1024, 1), (700, 2), (2048, 1), (513, 1)])
def test_large_J_population_round_trips_candidates(engine, J, nodes):
    """Large J: the search keeps its population in schedule order internally.  Candidates that enter (warm
    start, injected rows) and the incumbent that leaves are in the ABI's job-indexed encoding: a
    single-chain population returns exactly the warm candidate with the oracle's makespan, an injected
    better candidate replaces it, and greedy rounds never lose the incumbent."""
    T, _ = R.synth_table(J, 1, 8, seed=11, masked=False)
    engine.set_table(T, nodes=nodes)
    tab = R.reduce_table(R.canon_table(T, range(1, 9)))[0][:, None, :]
    rng = np.random.default_rng(J)
    def cand():
        k = rng.integers(0, 8, size=J)
        k = np.array([kk if np.isfinite(tab[j, 0, kk]) else int(np.argmin(tab[j, 0])) for j, kk in enumerate(k)])
        o = (k | (rng.integers(0, nodes, size=J) << 3)).astype(np.uint8)
        return o, rng.permutation(J).astype(np.uint16)
    o1, p1 = cand()
    mk1 = R.list_schedule(tab, o1, p1, True, np.float32, nodes=nodes)[0]
    engine.search_init(1, seed=1, reduced=True, t_start=0.0, t_end=0.0, warm=(o1, p1))
    assert engine.search_is_fused()
    bo, bp, bm, _ = engine.search_best()
    assert bm == mk1 and np.array_equal(bo, o1) and np.array_equal(bp, p1)
    # a clearly better candidate (every job on its fastest option, spread over the nodes) takes over
    o2 = (np.argmin(tab[:, 0, :], axis=1) | ((np.arange(J) % nodes) << 3)).astype(np.uint8)
    p2 = np.argsort(-tab[np.arange(J), 0, o2 & 7], kind="stable").astype(np.uint16)
    mk2 = R.list_schedule(tab, o2, p2, True, np.float32, nodes=nodes)[0]
    engine.search_init(64, seed=2, reduced=True, t_start=0.0, t_end=0.0, warm=(o1, p1))
    engine.search_inject(o2, p2, copies=8)
    bo, bp, bm, _ = engine.search_best()
    want = min(mk2, bm)
    assert bm <= mk2
    if bm == mk2:
        assert np.array_equal(bo, o2) and np.array_equal(bp, p2)
    engine.search_round(30)
    engine.search_resample()
    engine.search_round(30)
    bo, bp, bm3, _ = engine.search_best()
    assert bm3 <= want
    assert sorted(bp.tolist()) == list(range(J))
    assert R.list_schedule(tab, bo, bp, True, np.float32, nodes=nodes)[0] == bm3


@pytest.mark.parametrize("J,chains", [(1, 1), (2, 5), (3, 33), (7, 64)])
def test_tiny_problems_and_populations(J, chains):
    """Degenerate sizes: one task, populations smaller than a warp — the plan is still feasible and,
    being enumerable, optimal."""
    from saturn_b200 import solve
    rng = np.random.default_rng(J)
    tuples = [[(g, float(rng.uniform(10, 500)) / g ** 0.7) for g in (1, 4, 8)] for _ in range(J)]
    tasks = tasks_from_tuples(tuples)
    out = solve(tasks, None, chains=chains, rounds=40)
    mk = _check_plan(tasks, out)
    if J <= 3:
        tab, om = R.table_from_tuples(tuples)
        assert mk == pytest.approx(R.brute_force(tab, om, True)[0], rel=1e-9)
    assert solve([], None) [5] == 0.0


def test_solve_reaches_the_exhaustive_optimum_on_random_small_instances():
    """24 random instances (2-4 tasks, ragged option lists, 1 or 2 nodes): the plan returned by
    solve() is feasible under the reference's constraints and its makespan equals the exhaustive
    list-scheduling optimum — which is the reference MILP's optimum on every fixture."""
    from saturn_b200 import solve
    rng = np.random.default_rng(99)
    for trial in range(24):
        J = int(rng.integers(2, 5))
        nodes = int(rng.choice([1, 2]))
        tuples = []
        for _ in range(J):
            ks = sorted(rng.choice([1, 2, 3, 4, 6, 8], size=int(rng.integers(1, 4)), replace=False).tolist())
            base = float(rng.uniform(20, 900))
            tuples.append([(int(k), base * float(rng.uniform(1, 1.3)) / k ** float(rng.uniform(0.4, 1.0))) for k in ks])
        tasks = tasks_from_tuples(tuples)
        out = solve(tasks, None, chains=4096, rounds=48, nodes=nodes, seed=trial)
        sta, tga, bss, bna, boa, mk = out
        assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, mk) == [], trial
        tab, om = R.table_from_tuples(tuples)
        best = R.brute_force(tab, om, True, nodes=nodes)[0]
        assert mk == pytest.approx(best, rel=1e-9), (trial, J, nodes, tuples)


@pytest.mark.parametrize("J,S,nodes", [(64, 6, 1), (200, 1, 2), (600, 1, 1)])
def test_library_search_loop_equals_python_driver(engine, J, S, nodes):
    """sb_search_run (initialise, LPT seeds, rounds with resampling, stopping rules, all inside the library) and the
    Python driver used for the multi-GPU case issue the same device work: same seeds -> the same incumbent."""
    from saturn_b200.search import run_search
    T, valid = R.synth_table(J, S, 8, seed=21, masked=(S > 1))
    engine.set_table(T, nodes=nodes)
    reduced = S == 1
    kw = dict(chains=4096, rounds=48, seed=9, reduced=reduced, use_dist=False, record_history=True, exchange_every=8)
    a = run_search(engine, **kw)
    b = run_search(engine, _python_driver=True, **kw)
    assert a.makespan == b.makespan and np.array_equal(a.opt, b.opt) and np.array_equal(a.prio, b.prio)
    assert a.rounds == b.rounds == 48 and len(a.history) == len(b.history) == 7
    assert [h[2] for h in a.history] == [h[2] for h in b.history]
    tab = R.canon_table(T, range(1, 9))
    if reduced:
        tab = R.reduce_table(tab)[0][:, None, :]
    assert R.list_schedule(tab, a.opt, a.prio, True, np.float32, nodes=nodes)[0] == a.makespan
    # stopping rules: a target that the seeds already meet stops after the first group; patience stops a frozen search
    c = run_search(engine, chains=4096, rounds=400, seed=9, reduced=reduced, use_dist=False, target_makespan=a.makespan * 2,
                   exchange_every=8)
    assert c.rounds == 8
    d = run_search(engine, chains=64, rounds=4000, seed=9, reduced=reduced, use_dist=False, t_start=0.0, t_end=0.0,
                   patience=64, exchange_every=8)
    assert d.rounds < 4000


@pytest.mark.parametrize("J", [24, 300])
def test_plain_c_host_plans_through_the_abi(tmp_path, J):
    """examples/c_host.c — sb_create / sb_set_table / sb_search_run / sb_decode from C, no Python in the loop.
    The plan it prints is re-scored by the oracle on the table it prints: same makespan, feasible, and not
    worse than a longest-processing-time list schedule."""
    import subprocess
    from conftest import build_c_host
    out = subprocess.run([build_c_host(tmp_path), str(J), "11"], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    hdr = lines[0].split()
    Jp, S, G = int(hdr[1]), int(hdr[3]), int(hdr[5])
    assert Jp == J
    T = np.array(lines[1].split()[1:], dtype=np.float32).reshape(J, S, G)
    mk = float(lines[2].split()[1])
    assert float(lines[2].split()[3]) == mk                      # the decode re-derives the search's makespan
    opt = np.array(lines[3].split()[1:], dtype=np.uint8)
    prio = np.array(lines[4].split()[1:], dtype=np.int64)
    assert sorted(prio.tolist()) == list(range(J))
    tmin = R.reduce_table(R.canon_table(T, range(1, 9)))[0]
    got, start, mask, _ = R.list_schedule(tmin[:, None, :], opt, prio, True, np.float32)
    assert np.float32(got) == np.float32(mk)
    jobs = [l.split() for l in lines[5:5 + J]]
    assert [int(j[1]) for j in jobs] == list(range(J))
    k = np.array([int(j[5]) for j in jobs])
    assert np.array_equal(k, (opt & 7) + 1)
    assert np.array_equal(np.array([float(j[7]) for j in jobs], dtype=np.float32), np.asarray(start, dtype=np.float32))
    assert np.array_equal(np.array([int(j[9], 16) for j in jobs]), np.asarray(mask) & 0xff)
    rt = tmin[np.arange(J), opt & 7]
    ok, overlaps, _ = R.check_plan(start, mask, rt, k)
    assert ok and overlaps == 0
    # strategy = the arg-min strategy of the chosen GPU count (the profiler's min over executors)
    assert np.array_equal(np.array([int(j[3]) for j in jobs]), np.argmin(T[np.arange(J), :, k - 1], axis=1))
    lpt_order = np.argsort(-tmin[:, 7], kind="stable")
    lpt = R.list_schedule(tmin[:, None, :], np.full(J, 7, np.uint8), lpt_order, True, np.float32)[0]
    assert mk <= lpt


# ------------------------------------------------------------------------------------------ round 2
def test_solve_table_equals_solve_on_the_reduced_view(engine):
    """SURVEY §8f-3: the dense T[J][S][G] + mask entry gives the plan solve() gives on the task.strategies view
    the profiler would have built from the same trials (same seed, same population), plus the winning
    strategy per task."""
    from conftest import DuckTask
    from saturn_b200 import convert_into_comprehensible, solve, solve_table, strategies_from_table
    from saturn_b200 import solver as S
    J, Sx, G = 24, 4, 8
    T, valid = R.synth_table(J, Sx, G, seed=12)
    strategies = strategies_from_table(T, valid, executors=["e%d" % s for s in range(Sx)])
    tasks = [DuckTask("t%d" % j, strategies[j]) for j in range(J)]
    a = solve(tasks, None, chains=8192, rounds=40, seed=3, engine=engine)
    dev_a = S.last_stats["device_makespan"]
    b = solve_table(T, valid, chains=8192, rounds=40, seed=3, engine=engine)
    assert S.last_stats["device_makespan"] == dev_a
    assert b[5] == pytest.approx(a[5], rel=1e-12)
    assert a[0] == b[0] and a[1] == b[1] and a[2] == b[2] and a[3] == b[3] and a[4] == b[4]
    strategy = b[6]
    npt, tdd, starts = convert_into_comprehensible(tasks, b[2], b[4], b[1], b[3], b[0])
    for j, t in enumerate(tasks):
        g = t.selected_strategy.gpu_apportionment
        assert valid[j, strategy[j], g - 1]
        assert T[j, strategy[j], g - 1] == np.float32(t.selected_strategy.runtime)
        assert t.selected_strategy.executor == "e%d" % strategy[j]
    # a previous plan warm-starts the dense entry too, and a table without a mask treats sentinels as unusable
    c = solve_table(T, None, presolved=b[:6], chains=4096, rounds=10, seed=4, engine=engine)
    assert c[5] <= b[5] * (1 + 1e-6)
    for j in range(J):
        g = int(np.argmax(c[2][j])) + 1
        assert T[j, c[6][j], g - 1] < 1e6


@pytest.mark.parametrize("J,nodes", [(64, 1), (256, 1), (300, 1), (700, 1), (1024, 1), (64, 3), (700, 2)])
def test_initial_population_rows_are_valid(engine, J, nodes):
    """The shared-memory initialisation kernel (and the position-major one for large J) emits, for every
    chain, a permutation and existing table cells; two populations from one seed are identical and the
    incumbent of the freshly scored population decodes to its own makespan."""
    T, valid = R.synth_table(J, 3, 8, seed=J)
    engine.set_table(T, nodes=nodes)
    chains = 5000
    engine.search_init(chains, seed=9, chain_base=17, reduced=True)
    assert engine.search_validate() == 0
    o1, p1, mk1, key1 = engine.search_best()
    assert sorted(p1.tolist()) == list(range(J))
    engine.search_init(chains, seed=9, chain_base=17, reduced=True)
    o2, p2, mk2, key2 = engine.search_best()
    assert key1 == key2 and np.array_equal(o1, o2) and np.array_equal(p1, p2)
    dec = engine.decode(o1, p1, reduced=True)
    assert dec["makespan"] == mk1
    engine.search_init(chains, seed=10, chain_base=17, reduced=True)
    assert engine.search_best()[3] != key1
    engine.set_table(T)


@pytest.mark.parametrize("J", [256, 100, 300, 40, 700, 1024, 2100])
def test_incremental_rounds_equal_full_evaluation(engine, J):
    """Round 2: fused rounds score a proposal from the state snapshotted in front of the warp's window.
    (a) with the verify hook every incremental score is recomputed from position 0 on the device: none differs;
    (b) the search with snapshots and the search that scores the same windowed moves from position 0 walk
        the same chains: identical incumbent key, rows and history under a fixed seed;
    (c) the incumbent re-scores to its makespan in the oracle.
    J = 700 and up run the position-major kernel (both rows streamed; windows of whole 32-position blocks)."""
    from saturn_b200 import _lib
    from saturn_b200.search import run_search
    T, valid = R.synth_table(J, 3, 8, seed=100 + J)
    engine.set_table(T)
    # an explicit tournament cadence: the automatic one differs between the modes for position-major populations
    kw = dict(chains=9472, rounds=48, seed=11, reduced=True, use_dist=False, record_history=True, exchange_every=8,
              resample_every=4)
    a = run_search(engine, _extra_flags=_lib.HOOK_VERIFY_INCREMENTAL, **kw)
    assert engine.search_verify_count() == 0
    b = run_search(engine, _extra_flags=_lib.HOOK_NO_INCREMENTAL, **kw)
    c = run_search(engine, **kw)
    for x in (b, c):
        assert x.makespan == a.makespan and np.array_equal(x.opt, a.opt) and np.array_equal(x.prio, a.prio)
        assert [h[2] for h in x.history] == [h[2] for h in a.history]
    tab = R.canon_table(T, range(1, 9))
    tmin, _ = R.reduce_table(tab)
    assert float(R.list_schedule(tmin[:, None, :], c.opt, c.prio, True, np.float32)[0]) == c.makespan
    assert c.history[-1][2] < c.history[0][2] or J <= 40
    # the round-1 move generator (no windows) reaches a comparable plan: the windows cost no quality
    d = run_search(engine, _extra_flags=_lib.HOOK_ROUND1_MOVES, **kw)
    assert c.makespan <= d.makespan * 1.01
