"""GPU: the worst- and mean-makespan objectives over runtime scenarios (SB_FLAG_WORST_MAKESPAN, SB_FLAG_MEAN_MAKESPAN;
solve(objective="worst_makespan" | "mean_makespan", scenarios=...)) — every route that scores them (the generic kernel
on job-indexed rows, the position-major kernel on rows by position and after the device re-order) bit for bit against
oracle/ref_scenarios.py, sb_eval_scenarios' per-scenario makespans, K = 1 with unit factors against the makespan
kernels, the search population after every kind of round, the exhaustive optima of the fixtures through solve() and
solve_table(), orchestrate(), several devices, and every refusal of the C ABI."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from conftest import DuckTask, tasks_from_tuples
from oracle import ref_eval as R, ref_scenarios as SC
from saturn_b200.engine import opt_by_position, random_candidates

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
KEY_MAX = 2 ** 63 - 1
OBJS = ("worst_makespan", "mean_makespan")


def _factors(K, J, seed):
    return np.random.default_rng(seed).lognormal(0.0, 0.3, size=(K, J)).astype(np.float32)


def _key_of(ref, id_base):
    i = int(np.argmin(ref))
    return (int(ref[i:i + 1].view(np.uint32)[0]) << 32) | (id_base + i)


def _eval(engine, opt, prio, objective, **kw):
    key = torch.full((1,), KEY_MAX, dtype=torch.int64, device=engine.device)
    got = engine.eval(opt, prio, objective=objective, best_key=key, id_base=7, **kw)
    torch.cuda.synchronize()
    return got.cpu().numpy(), int(key.item()), engine.last_eval_path()


def _nodes_candidates(engine, J, B, nodes, seed):
    """A one-strategy table (so that the scenario tables of every size here fit in shared memory, and several nodes
    read it as the reduced table) and candidates; with several nodes the opt bytes carry a node."""
    T, valid = R.synth_table(J, 1, 8, seed=seed, masked=nodes == 1)
    engine.set_table(T, nodes=nodes)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=seed + 1, nodes=nodes)
    return tab, opt, prio


@pytest.mark.parametrize("J", [5, 64, 256, 300])
@pytest.mark.parametrize("K", [1, 3, 8])
@pytest.mark.parametrize("nodes", [1, 2])
def test_eval_routes_bit_exact(engine, J, K, nodes):
    """sb_eval under both flags, integer starts on and off, release dates on and off: the generic kernel (job-indexed
    rows, path 0) and the position-major kernel (rows by position, path 5; job-indexed rows re-ordered on the device,
    path 9) give the oracle's fp32 score bit for bit, and the arg-min key; u16 priorities at J = 300."""
    B = 1500 if J <= 256 else 600
    tab, opt, prio = _nodes_candidates(engine, J, B, nodes, seed=J + K)
    reduced = nodes > 1
    f = _factors(K, J, J * K)
    engine.set_scenarios(f)
    r = np.random.default_rng(J).uniform(-50.0, 4000.0, size=J).astype(np.float32)
    opt_np, prio_np = opt.cpu().numpy(), prio.cpu().numpy()
    aligned = opt.stride(0) % 32 == 0
    for rel in (None, r):
        engine.set_release(rel)
        for ints in (True, False):
            for obj in OBJS:
                ref = SC.evaluate(tab, opt_np, prio_np, f, obj, rel, ints, np.float32, nodes)
                assert (ref > 0).all()
                runs = [({}, 0), ({"_force_generic": True}, 0)]
                if aligned:
                    runs.append(({"_reorder": True}, 9))
                for kw, path in runs:
                    got, key, p = _eval(engine, opt, prio, obj, integer_starts=ints, reduced=reduced, **kw)
                    assert p == path, (kw, p)
                    assert got.tobytes() == ref.tobytes(), (obj, ints, rel is not None, kw)
                    assert key == _key_of(ref, 7)
                obp = opt_by_position(opt, prio)
                got, key, p = _eval(engine, obp, prio, obj, integer_starts=ints, reduced=reduced, by_position=True)
                assert p == 5 and got.tobytes() == ref.tobytes() and key == _key_of(ref, 7)
                host = engine.eval_host(opt.cpu(), prio.cpu(), integer_starts=ints, reduced=reduced, objective=obj)
                assert host.numpy().tobytes() == ref.tobytes()
    engine.set_release(None)


@pytest.mark.parametrize("nodes", [1, 2])
@pytest.mark.parametrize("released", [False, True])
def test_eval_full_makespans_and_decode(engine, nodes, released):
    """sb_eval_scenarios returns every scenario's makespan M_k as the oracle does, and the score; sb_eval_full and
    sb_decode report the score with the start times and slot masks of the nominal schedule."""
    J, B, K = 48, 700, 5
    tab, opt, prio = _nodes_candidates(engine, J, B, nodes, seed=77)
    reduced = nodes > 1
    f = _factors(K, J, 78)
    engine.set_scenarios(f)
    rel = np.random.default_rng(3).uniform(0.0, 3000.0, size=J).astype(np.float32) if released else None
    engine.set_release(rel)
    opt_np, prio_np = opt.cpu().numpy(), prio.cpu().numpy()
    for ints in (True, False):
        nominal, nstart, nmask = engine.eval_full(opt, prio, integer_starts=ints, reduced=reduced)
        for obj in OBJS:
            ref, M = SC.evaluate(tab, opt_np, prio_np, f, obj, rel, ints, np.float32, nodes, want_makespans=True)
            score, mks = engine.eval_scenarios(opt, prio, integer_starts=ints, reduced=reduced, objective=obj)
            assert score.cpu().numpy().tobytes() == ref.tobytes()
            assert mks.cpu().numpy().tobytes() == M.tobytes()
            full, start, mask = engine.eval_full(opt, prio, integer_starts=ints, reduced=reduced, objective=obj)
            assert full.cpu().numpy().tobytes() == ref.tobytes()
            assert torch.equal(start, nstart) and torch.equal(mask, nmask)
            dec = engine.decode(opt_np[3], prio_np[3], integer_starts=ints, reduced=reduced, objective=obj)
            assert dec["makespan"] == float(ref[3])
            assert np.array_equal(dec["start"], nstart[3].cpu().numpy())
    engine.set_release(None)


@pytest.mark.parametrize("ints", [True, False])
def test_one_unit_scenario_is_the_makespan_path(engine, ints):
    """K = 1 with f = 1: both flags score exactly what the makespan kernels score, on every route, and
    sb_eval_scenarios' single makespan is the slot-exact makespan."""
    J, B = 128, 3000
    T, valid = R.synth_table(J, 4, 8, seed=5)
    engine.set_table(T)
    opt, prio = random_candidates(engine, B, valid, seed=6)
    engine.set_scenarios(np.ones((1, J), np.float32))
    mk, _, _ = _eval(engine, opt, prio, "makespan", integer_starts=ints)
    full, _s, _m = engine.eval_full(opt, prio, integer_starts=ints)
    for obj in OBJS:
        got, _, _ = _eval(engine, opt, prio, obj, integer_starts=ints)
        assert got.tobytes() == mk.tobytes()
        got, _, _ = _eval(engine, opt_by_position(opt, prio), prio, obj, integer_starts=ints, by_position=True)
        assert got.tobytes() == mk.tobytes()
        score, mks = engine.eval_scenarios(opt, prio, integer_starts=ints, objective=obj)
        assert score.cpu().numpy().tobytes() == mk.tobytes() and torch.equal(mks[:, 0], full)


def test_refusals(engine):
    """sb_set_scenarios refuses K outside 1..8, a J that is not the table's and a factor <= 0, NaN or inf (SB_ERR_ARG)
    and comes before any table (SB_ERR_STATE); either flag without scenarios is SB_ERR_STATE, both flags or either
    with another objective flag SB_ERR_ARG, the alternate shape SB_ERR_UNSUPPORTED, and scenario tables beyond one
    CTA's shared memory SB_ERR_UNSUPPORTED, refused on the host.  sb_set_table drops the scenarios; release dates
    combine with both flags."""
    from saturn_b200 import _lib
    from saturn_b200.engine import Engine
    J = 32
    T, valid = R.synth_table(J, 2, 8, seed=1)
    fresh = Engine(0)
    f = np.ones((2, J), np.float32)
    assert fresh._lib.sb_set_scenarios(fresh._h, C.c_void_p(f.ctypes.data), 2, J) == -3
    fresh.close()
    engine.set_table(T)
    opt, prio = random_candidates(engine, 64, valid, seed=1)
    out = torch.empty(64, dtype=torch.float32, device=engine.device)
    WM, MM = _lib.FLAG_WORST_MAKESPAN, _lib.FLAG_MEAN_MAKESPAN

    def raw(flags):
        return engine._lib.sb_eval(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 64, J, flags,
                                   C.c_void_p(out.data_ptr()), None, 0)

    def set_f(arr, K, JJ=J):
        a = np.ascontiguousarray(arr, dtype=np.float32)
        return engine._lib.sb_set_scenarios(engine._h, C.c_void_p(a.ctypes.data), K, JJ)
    try:
        assert raw(WM) == -3 and raw(MM) == -3
        assert "sb_set_scenarios" in engine._lib.sb_last_error().decode()
        p = _lib.SearchParams(seed=1, chains=256, flags=_lib.FLAG_REDUCED | WM, t_start=0.01, t_end=1e-4,
                              total_rounds=4)
        assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -3
        for arr, K, JJ in ((np.ones((9, J)), 9, J), (np.ones((1, J)), 0, J), (np.ones((2, J + 1)), 2, J + 1)):
            assert set_f(arr, K, JJ) == -1
        for bad in (0.0, -1.0, float("nan"), float("inf")):
            arr = np.ones((3, J))
            arr[2, 5] = bad
            assert set_f(arr, 3) == -1, bad
        # device factors are accepted too
        dev = torch.ones((2, J), dtype=torch.float32, device=engine.device)
        assert engine._lib.sb_set_scenarios(engine._h, C.c_void_p(dev.data_ptr()), 2, J) == 0
        assert raw(WM) == 0 and raw(MM) == 0
        assert raw(WM | _lib.FLAG_RELEASE) == -3
        engine.set_release(np.arange(J, dtype=np.float32))
        assert raw(WM | _lib.FLAG_RELEASE) == 0 and raw(MM | _lib.FLAG_RELEASE) == 0
        for other in (MM, _lib.FLAG_SUM_COMPLETION, _lib.FLAG_WEIGHTED, _lib.FLAG_DUE, _lib.FLAG_MAX_LATENESS,
                      _lib.FLAG_LATE_COUNT, _lib.FLAG_MAX_TARDINESS, _lib.FLAG_SQUARED, _lib.FLAG_LATE_PENALTY,
                      _lib.FLAG_COMPLETION_PENALTY, _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE):
            assert raw(WM | other) == -1, other
            assert raw(MM | other if other != MM else MM | WM) == -1, other
        p.flags = _lib.FLAG_REDUCED | WM | MM
        assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -1
        assert raw(WM | _lib.FLAG_ALT_WARPSCAN) == -4 and raw(MM | _lib.FLAG_ALT_WARPSCAN) == -4
        score = torch.empty(64, dtype=torch.float32, device=engine.device)
        assert engine._lib.sb_eval_scenarios(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 64,
                                             J, 0, C.c_void_p(score.data_ptr()), C.c_void_p(out.data_ptr())) == -1
        engine.set_table(T)                                                          # drops the scenarios
        assert raw(WM) == -3 and raw(0) == 0
        # J = 256 with 8 strategies: 8 full tables are 512 KB, refused before any launch; the reduced tables fit
        J2 = 256
        T2, valid2 = R.synth_table(J2, 8, 8, seed=2)
        engine.set_table(T2)
        o2, p2 = random_candidates(engine, 64, valid2, seed=2)
        assert set_f(np.ones((8, J2)), 8, J2) == 0
        out2 = torch.empty(64, dtype=torch.float32, device=engine.device)
        rc = engine._lib.sb_eval(engine._h, C.c_void_p(o2.data_ptr()), C.c_void_p(p2.data_ptr()), 64, J2, WM,
                                 C.c_void_p(out2.data_ptr()), None, 0)
        assert rc == -4 and "shared memory" in engine._lib.sb_last_error().decode()
        p.flags = WM
        assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -4
        p.flags = _lib.FLAG_REDUCED | WM
        assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == 0
    finally:
        engine.set_table(T)


@pytest.mark.parametrize("J,nodes", [(40, 1), (256, 1), (300, 1), (64, 2)])
@pytest.mark.parametrize("released", [False, True])
def test_population_after_every_kind_of_round(engine, J, nodes, released):
    """After init, seeding and rounds of 1, 3, 16 and 17 — position-major (the layout the library picks) and unfused
    propose / evaluate / accept rounds — sb_search_validate finds no bad row and every chain's stored score is the
    oracle's score of its rows; the search result re-scores to the reported value."""
    from saturn_b200.search import run_search
    T, valid = R.synth_table(J, 1 if nodes > 1 else 3, 8, seed=200 + J, masked=nodes == 1)
    tmin = R.reduce_table(R.canon_table(T, range(1, 9)))[0][:, None, :]
    engine.set_table(T, nodes=nodes)
    K = 4
    f = _factors(K, J, J)
    engine.set_scenarios(f)
    horizon = float(np.nanmin(np.where(np.isfinite(tmin), tmin, np.nan), axis=2).sum()) / 8
    rel = (np.random.default_rng(J).uniform(0.0, 0.5, size=J) * horizon).astype(np.float32) if released else None
    engine.set_release(rel)
    try:
        for obj in OBJS:
            res = run_search(engine, chains=4096, rounds=24, seed=11, reduced=True, use_dist=False, exchange_every=8,
                             resample_every=4, objective=obj, t_start=0.05, t_end=0.01)
            assert sorted(res.prio.tolist()) == list(range(J))
            ref = SC.evaluate(tmin, res.opt[None], res.prio[None], f, obj, rel, True, np.float32, nodes)
            assert float(ref[0]) == res.makespan
            layouts = set()
            for no_fused in (False, True):
                engine.search_init(2048, seed=3, reduced=True, t_start=0.01, t_end=1e-4, total_rounds=40,
                                   objective=obj, _no_fused=no_fused)

                def check(what):
                    assert engine.search_validate() == 0, what
                    opt, prio, score, layout = engine.debug_search_population()
                    want = SC.evaluate(tmin, opt, prio, f, obj, rel, True, np.float32, nodes)
                    assert score.tobytes() == want.tobytes(), what
                    return layout
                check("init")
                engine.search_seed_lpt()
                check("seeds")
                for n in (1, 3, 16, 17):
                    engine.search_round(n)
                    layouts.add(check("rounds %d, no_fused %s" % (n, no_fused)))
            assert layouts == {0, 2}
    finally:
        engine.set_release(None)


def _cases():
    with open(os.path.join(HERE, "golden", "scenario_cases.json")) as f:
        return json.load(f)["cases"]


def _plan(tasks, out):
    sta, tga, bss, bna, boa, mk = out
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, mk) == []
    plan = R.plan_from_arrays(tuples, sta, tga, bss, bna)
    # the slot masks are per node (plan_from_arrays returns the node last): check each node's tasks on their own
    for n in sorted({p[5] for p in plan}):
        on = [p for p in plan if p[5] == n]
        ok, ov, _ = R.check_plan([p[0] for p in on], [p[1] for p in on], [p[2] for p in on], [p[3] for p in on])
        assert ok and ov == 0, n


def test_solve_reaches_the_exhaustive_optimum():
    """Every fixture instance under both objectives: solve() returns a plan that passes check_plan and the MILP's
    constraints on the nominal table, whose fp32 device score is the fixture's fp32 exhaustive optimum; last_stats'
    float64 rescore matches the oracle's float64 makespans of that plan; solve_table on the same table returns a plan
    with the same score.  Scenarios go in as a sequence for solve_table and as a mapping for solve()."""
    from saturn_b200 import solve_table
    from saturn_b200 import solver as S
    cases = _cases()
    for i, rec in enumerate(cases):
        tuples = rec["gpu_time_tuples"]
        tasks = tasks_from_tuples(tuples)
        J = len(tasks)
        fT = np.asarray(rec["factors"], dtype=np.float64).T          # [J][K]
        for obj in OBJS:
            kw = {"objective": obj, "release": rec["release"], "nodes": rec["nodes"]}
            out = S.solve(tasks, None, chains=4096, rounds=60, seed=i,
                          scenarios={t: list(fT[j]) for j, t in enumerate(tasks)}, **kw)
            _plan(tasks, out)
            st = dict(S.last_stats)
            assert st["device_makespan"] == rec[obj + "_f32"]["score"], (rec["name"], obj)
            assert len(st["scenario_makespans"]) == len(rec["factors"])
            assert st["worst_makespan"] == max(st["scenario_makespans"])
            assert st["mean_makespan"] == pytest.approx(sum(st["scenario_makespans"]) / len(rec["factors"]))
            assert out[5] == pytest.approx(st["makespan"])
            T = np.full((J, 1, 8), np.inf, np.float32)
            for j, tup in enumerate(tuples):
                for g, rt in tup:
                    T[j, 0, int(g) - 1] = rt
            solve_table(T, np.isfinite(T), chains=4096, rounds=60, seed=i, scenarios=fT, **kw)
            assert S.last_stats["device_makespan"] == rec[obj + "_f32"]["score"], (rec["name"], obj)


def test_last_stats_is_a_float64_rescore():
    """On a 64-task set with log-normal factors, last_stats' scenario makespans are the float64 list schedule of the
    plan's options and order on f * rt (integer starts), within fp32 rounding of the device's score."""
    from saturn_b200 import solver as S
    from saturn_b200.solver import strategies_from_table
    from saturn_b200.synth import synth_table
    J, K = 64, 6
    T, valid = synth_table(J, 4, 8, seed=12)
    st = strategies_from_table(T, valid)
    tasks = [DuckTask("t%d" % j, st[j]) for j in range(J)]
    fT = np.random.default_rng(13).lognormal(0.0, 0.3, size=(J, K))
    for obj in OBJS:
        S.solve(tasks, None, chains=8192, rounds=60, seed=2, objective=obj, scenarios=fT)
        s = S.last_stats
        score = max(s["scenario_makespans"]) if obj == "worst_makespan" else sum(s["scenario_makespans"])
        assert score == pytest.approx(s["device_makespan"], rel=1e-5)
        assert s["worst_makespan"] == max(s["scenario_makespans"])
        assert s["mean_makespan"] == pytest.approx(sum(s["scenario_makespans"]) / K, rel=1e-12)


def test_orchestrate_runs_in_simulated_time():
    """orchestrate() with a scenarios mapping keyed by Task runs every task to completion."""
    from saturn_b200 import orchestrate
    rng = np.random.default_rng(9)
    tuples = [[(g, float(rng.uniform(800, 5000)) / g ** 0.8) for g in (1, 2, 4, 8)] for _ in range(8)]
    tasks = tasks_from_tuples(tuples)
    for t in tasks:
        t.total_batches = 200
    kw = {"chains": 4096, "rounds": 25, "objective": "mean_makespan",
          "scenarios": {t: [1.0, 1.0 + 0.1 * i, 0.8] for i, t in enumerate(tasks)}}
    orchestrate(tasks, interval=1000, solver_kwargs=kw, max_intervals=50)
    assert all(t.total_batches == 0 for t in tasks)


def test_multiple_devices_give_a_valid_plan():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from saturn_b200 import solver as S
    rec = _cases()[2]
    tasks = tasks_from_tuples(rec["gpu_time_tuples"])
    out = S.solve(tasks, None, chains=2048, rounds=40, seed=1, devices=2, objective="worst_makespan",
                  scenarios=np.asarray(rec["factors"]).T, release=rec["release"])
    _plan(tasks, out)
    assert S.last_stats["devices"] == 2
    assert S.last_stats["device_makespan"] == rec["worst_makespan_f32"]["score"]
