"""GPU: the worst- and mean-tardiness objectives over runtime scenarios (SB_FLAG_WORST_TARDINESS,
SB_FLAG_MEAN_TARDINESS; solve(objective="worst_tardiness" | "mean_tardiness" | "worst_completion" |
"mean_completion", scenarios=...)) — every route that scores them (the generic kernel on job-indexed rows, the
position-major kernel on rows by position and after the device re-order, sb_eval_host) bit for bit against
oracle/ref_scenario_tardiness.py, sb_eval_scenarios' per-scenario totals, K = 1 with unit factors against the
tardiness kernels and with d = 0 against the completion kernels, the search population after every kind of round, the
exhaustive optima of the fixtures through solve() and solve_table(), orchestrate(), several devices, and every refusal
of the C ABI."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from conftest import DuckTask, tasks_from_tuples
from oracle import ref_eval as R, ref_scenario_tardiness as ST
from saturn_b200.engine import opt_by_position, random_candidates

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
KEY_MAX = 2 ** 63 - 1
FORMS = ("worst_tardiness", "mean_tardiness")       # the oracle's names of the two device forms


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


def _engine_name(form, weighted):
    return ("weighted_" if weighted else "") + form


def _nodes_candidates(engine, J, B, nodes, seed):
    """A one-strategy table (so that the scenario tables of every size here fit in shared memory, and several nodes
    read it as the reduced table) and candidates; with several nodes the opt bytes carry a node."""
    T, valid = R.synth_table(J, 1, 8, seed=seed, masked=nodes == 1)
    engine.set_table(T, nodes=nodes)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=seed + 1, nodes=nodes)
    return tab, opt, prio


def _horizon(tab, nodes=1):
    tmin = R.reduce_table(tab)[0]
    return float(np.nanmin(np.where(np.isfinite(tmin), tmin, np.nan), axis=1).sum()) / (8 * nodes)


def _per_job(engine, J, seed, horizon):
    rng = np.random.default_rng(seed)
    d = np.round(rng.uniform(0.0, horizon, size=J)).astype(np.float32)
    w = rng.uniform(0.25, 4.0, size=J).astype(np.float32)
    engine.set_due(d)
    engine.set_weights(w)
    return d, w


@pytest.fixture
def scen_engine(engine):
    """The session engine, its release dates, due dates and weights cleared again after each test."""
    yield engine
    engine.set_release(None)


@pytest.mark.parametrize("J", [5, 64, 256, 300])
@pytest.mark.parametrize("K", [1, 3, 8])
@pytest.mark.parametrize("nodes", [1, 2])
def test_eval_routes_bit_exact(scen_engine, J, K, nodes):
    """sb_eval under both flags, weighted and unweighted, integer starts on and off, release dates on and off: the
    generic kernel (job-indexed rows, path 0), the position-major kernel (rows by position, path 5; job-indexed rows
    re-ordered on the device, path 9) and sb_eval_host give the oracle's fp32 score bit for bit, and the arg-min key;
    u16 priorities at J = 300."""
    engine = scen_engine
    B = 1500 if J <= 256 else 600
    tab, opt, prio = _nodes_candidates(engine, J, B, nodes, seed=J + K)
    reduced = nodes > 1
    f = _factors(K, J, J * K)
    engine.set_scenarios(f)
    d, w = _per_job(engine, J, J + 1, _horizon(tab, nodes))
    r = np.random.default_rng(J).uniform(-50.0, 4000.0, size=J).astype(np.float32)
    opt_np, prio_np = opt.cpu().numpy(), prio.cpu().numpy()
    aligned = opt.stride(0) % 32 == 0
    for rel in (None, r):
        engine.set_release(rel)
        for ints in (True, False):
            for form in FORMS:
                for weighted in (False, True):
                    name = _engine_name(form, weighted)
                    ref, _ = ST.c_evaluate(tab, opt_np, prio_np, f, form, d, w if weighted else None, rel, ints,
                                           nodes)
                    assert (ref > 0).any()
                    runs = [({}, 0), ({"_force_generic": True}, 0)]
                    if aligned:
                        runs.append(({"_reorder": True}, 9))
                    for kw, path in runs:
                        got, key, p = _eval(engine, opt, prio, name, integer_starts=ints, reduced=reduced, **kw)
                        assert p == path, (kw, p)
                        assert got.tobytes() == ref.tobytes(), (name, ints, rel is not None, kw)
                        assert key == _key_of(ref, 7)
                    obp = opt_by_position(opt, prio)
                    got, key, p = _eval(engine, obp, prio, name, integer_starts=ints, reduced=reduced,
                                        by_position=True)
                    assert p == 5 and got.tobytes() == ref.tobytes() and key == _key_of(ref, 7)
                    host = engine.eval_host(opt.cpu(), prio.cpu(), integer_starts=ints, reduced=reduced,
                                            objective=name)
                    assert host.numpy().tobytes() == ref.tobytes()


@pytest.mark.parametrize("nodes", [1, 2])
@pytest.mark.parametrize("released", [False, True])
def test_eval_full_totals_and_decode(scen_engine, nodes, released):
    """sb_eval_scenarios returns every scenario's total S_k as the oracle does, and the score; sb_eval_full and
    sb_decode report the score with the start times and slot masks of the nominal schedule."""
    engine = scen_engine
    J, B, K = 48, 700, 5
    tab, opt, prio = _nodes_candidates(engine, J, B, nodes, seed=77)
    reduced = nodes > 1
    f = _factors(K, J, 78)
    engine.set_scenarios(f)
    d, w = _per_job(engine, J, 79, _horizon(tab, nodes))
    rel = np.random.default_rng(3).uniform(0.0, 3000.0, size=J).astype(np.float32) if released else None
    engine.set_release(rel)
    opt_np, prio_np = opt.cpu().numpy(), prio.cpu().numpy()
    for ints in (True, False):
        nominal, nstart, nmask = engine.eval_full(opt, prio, integer_starts=ints, reduced=reduced)
        for form in FORMS:
            for weighted in (False, True):
                name = _engine_name(form, weighted)
                ref, S = ST.evaluate(tab, opt_np, prio_np, f, form, d, w if weighted else None, rel, ints,
                                     np.float32, nodes, want_totals=True)
                score, tot = engine.eval_scenarios(opt, prio, integer_starts=ints, reduced=reduced, objective=name)
                assert score.cpu().numpy().tobytes() == ref.tobytes()
                assert tot.cpu().numpy().tobytes() == S.tobytes()
                full, start, mask = engine.eval_full(opt, prio, integer_starts=ints, reduced=reduced, objective=name)
                assert full.cpu().numpy().tobytes() == ref.tobytes()
                assert torch.equal(start, nstart) and torch.equal(mask, nmask)
                dec = engine.decode(opt_np[3], prio_np[3], integer_starts=ints, reduced=reduced, objective=name)
                assert dec["makespan"] == float(ref[3])
                assert np.array_equal(dec["start"], nstart[3].cpu().numpy())


@pytest.mark.parametrize("ints", [True, False])
@pytest.mark.parametrize("released", [False, True])
def test_one_unit_scenario_and_zero_due_dates(scen_engine, ints, released):
    """K = 1 with f = 1: both flags score what the tardiness / weighted-tardiness kernels score; with every due date
    +0 what the completion / weighted-completion kernels score — bit for bit on every route (generic, position-major,
    re-ordered, slot-exact), release dates negative and positive."""
    engine = scen_engine
    J, B = 128, 3000
    T, valid = R.synth_table(J, 1, 8, seed=5)
    engine.set_table(T)
    tab = R.canon_table(T, range(1, 9))
    opt, prio = random_candidates(engine, B, valid, seed=6)
    engine.set_scenarios(np.ones((1, J), np.float32))
    d, _ = _per_job(engine, J, 7, _horizon(tab))
    rel = np.random.default_rng(8).uniform(-500.0, 3000.0, size=J).astype(np.float32) if released else None
    engine.set_release(rel)
    obp = opt_by_position(opt, prio)
    for due, nominal in ((d, "tardiness"), (np.zeros(J, np.float32), "completion")):
        engine.set_due(due)
        for weighted in (False, True):
            base = ("weighted_" if weighted else "") + nominal
            want, _, _ = _eval(engine, opt, prio, base, integer_starts=ints)
            wfull, _s, _m = engine.eval_full(opt, prio, integer_starts=ints, objective=base)
            assert wfull.cpu().numpy().tobytes() == want.tobytes()
            for form in FORMS:
                name = _engine_name(form, weighted)
                for kw in ({}, {"_reorder": True}):
                    got, _, _ = _eval(engine, opt, prio, name, integer_starts=ints, **kw)
                    assert got.tobytes() == want.tobytes(), (base, name, kw)
                got, _, _ = _eval(engine, obp, prio, name, integer_starts=ints, by_position=True)
                assert got.tobytes() == want.tobytes(), (base, name)
                score, tot = engine.eval_scenarios(opt, prio, integer_starts=ints, objective=name)
                assert score.cpu().numpy().tobytes() == want.tobytes() and torch.equal(tot[:, 0], wfull)


def test_refusals(scen_engine):
    """Either flag without scenarios, due dates or (with SB_FLAG_WEIGHTED) weights is SB_ERR_STATE; both flags, either
    without SB_FLAG_SUM_COMPLETION | SB_FLAG_DUE, or either with another objective modifier or a makespan scenario flag
    is SB_ERR_ARG; the alternate shape and scenario tables beyond one CTA's shared memory SB_ERR_UNSUPPORTED, refused
    on the host.  The makespan pair keeps its refusals; release dates combine with both flags; sb_set_table drops the
    scenarios."""
    from saturn_b200 import _lib
    engine = scen_engine
    J = 32
    T, valid = R.synth_table(J, 2, 8, seed=1)
    engine.set_table(T)
    opt, prio = random_candidates(engine, 64, valid, seed=1)
    out = torch.empty(64, dtype=torch.float32, device=engine.device)
    base = _lib.FLAG_SUM_COMPLETION | _lib.FLAG_DUE
    WT, MT = _lib.FLAG_WORST_TARDINESS, _lib.FLAG_MEAN_TARDINESS
    WM, MM = _lib.FLAG_WORST_MAKESPAN, _lib.FLAG_MEAN_MAKESPAN

    def raw(flags):
        return engine._lib.sb_eval(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 64, J, flags,
                                   C.c_void_p(out.data_ptr()), None, 0)

    def set_f(K, JJ=J):
        a = np.ones((K, JJ), dtype=np.float32)
        return engine._lib.sb_set_scenarios(engine._h, C.c_void_p(a.ctypes.data), K, JJ)
    try:
        # the state checks, in order: due dates, weights, scenarios
        for flag in (WT, MT):
            assert raw(base | flag) == -3
            assert "sb_set_due" in engine._lib.sb_last_error().decode()
        engine.set_due(np.full(J, 500.0, np.float32))
        assert raw(base | WT | _lib.FLAG_WEIGHTED) == -3
        assert "sb_set_weights" in engine._lib.sb_last_error().decode()
        engine.set_weights(np.ones(J, np.float32))
        for flag in (WT, MT):
            assert raw(base | flag) == -3 and raw(base | flag | _lib.FLAG_WEIGHTED) == -3
            assert "sb_set_scenarios" in engine._lib.sb_last_error().decode()
        p = _lib.SearchParams(seed=1, chains=256, flags=_lib.FLAG_REDUCED | base | WT, t_start=0.01, t_end=1e-4,
                              total_rounds=4)
        assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -3
        assert set_f(2) == 0
        for flag in (WT, MT):
            assert raw(base | flag) == 0 and raw(base | flag | _lib.FLAG_WEIGHTED) == 0
            assert raw(base | flag | _lib.FLAG_RELEASE) == -3
        engine.set_release(np.arange(J, dtype=np.float32))
        for flag in (WT, MT):
            assert raw(base | flag | _lib.FLAG_RELEASE) == 0
            # not without SUM_COMPLETION | DUE
            for partial in (0, _lib.FLAG_SUM_COMPLETION, _lib.FLAG_DUE, _lib.FLAG_WEIGHTED,
                            _lib.FLAG_SUM_COMPLETION | _lib.FLAG_WEIGHTED):
                assert raw(partial | flag) == -1, (flag, partial)
            for other in (_lib.FLAG_LATE_COUNT, _lib.FLAG_MAX_TARDINESS, _lib.FLAG_SQUARED, _lib.FLAG_LATE_PENALTY,
                          _lib.FLAG_COMPLETION_PENALTY, _lib.FLAG_MAX_LATENESS, WM, MM):
                assert raw(base | flag | other) == -1, (flag, other)
            assert raw(base | flag | _lib.FLAG_ALT_WARPSCAN) == -4
        assert raw(base | WT | MT) == -1
        p.flags = _lib.FLAG_REDUCED | base | WT | MT
        assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -1
        # the makespan pair's refusals are unchanged
        assert raw(WM | base) == -1 and raw(MM | base) == -1 and raw(WM | MM) == -1
        assert raw(WM) == 0 and raw(MM) == 0
        assert raw(WM | _lib.FLAG_ALT_WARPSCAN) == -4
        score = torch.empty(64, dtype=torch.float32, device=engine.device)
        assert engine._lib.sb_eval_scenarios(engine._h, C.c_void_p(opt.data_ptr()), C.c_void_p(prio.data_ptr()), 64,
                                             J, base, C.c_void_p(score.data_ptr()), C.c_void_p(out.data_ptr())) == -1
        engine.set_table(T)                                                          # drops the scenarios
        engine.set_due(np.full(J, 500.0, np.float32))
        assert raw(base | WT) == -3 and raw(base) == 0
        # J = 256: 8 full tables of 8 strategies are refused before any launch, naming the limit; the reduced fit
        J2 = 256
        T2, valid2 = R.synth_table(J2, 8, 8, seed=2)
        engine.set_table(T2)
        engine.set_due(np.full(J2, 500.0, np.float32))
        o2, p2 = random_candidates(engine, 64, valid2, seed=2)
        o2r = (o2 & 7).contiguous()                     # the reduced table's opt bytes: k - 1
        assert set_f(8, J2) == 0
        out2 = torch.empty(64, dtype=torch.float32, device=engine.device)
        for flag in (WT, MT):
            rc = engine._lib.sb_eval(engine._h, C.c_void_p(o2.data_ptr()), C.c_void_p(p2.data_ptr()), 64, J2,
                                     base | flag, C.c_void_p(out2.data_ptr()), None, 0)
            assert rc == -4 and "shared memory" in engine._lib.sb_last_error().decode()
            rc = engine._lib.sb_eval(engine._h, C.c_void_p(o2r.data_ptr()), C.c_void_p(p2.data_ptr()), 64, J2,
                                     base | flag | _lib.FLAG_REDUCED, C.c_void_p(out2.data_ptr()), None, 0)
            assert rc == 0
        torch.cuda.synchronize()
        p.flags = base | WT
        assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == -4
        p.flags = _lib.FLAG_REDUCED | base | MT
        assert engine._lib.sb_search_init(engine._h, C.byref(p), None, None) == 0
    finally:
        engine.set_table(T)


@pytest.mark.parametrize("J,nodes", [(40, 1), (256, 1), (300, 1), (64, 2)])
@pytest.mark.parametrize("released", [False, True])
def test_population_after_every_kind_of_round(scen_engine, J, nodes, released):
    """After init, seeding and rounds of 1, 3, 16 and 17 — position-major (the layout the library picks) and unfused
    propose / evaluate / accept rounds — sb_search_validate finds no bad row and every chain's stored score is the
    oracle's score of its rows; the search result re-scores to the reported value."""
    from saturn_b200.search import run_search
    engine = scen_engine
    T, valid = R.synth_table(J, 1 if nodes > 1 else 3, 8, seed=200 + J, masked=nodes == 1)
    tmin = R.reduce_table(R.canon_table(T, range(1, 9)))[0][:, None, :]
    engine.set_table(T, nodes=nodes)
    K = 4
    f = _factors(K, J, J)
    engine.set_scenarios(f)
    horizon = float(np.nanmin(np.where(np.isfinite(tmin), tmin, np.nan), axis=2).sum()) / 8
    d, w = _per_job(engine, J, J + 3, 2 * horizon)
    rel = (np.random.default_rng(J).uniform(0.0, 0.5, size=J) * horizon).astype(np.float32) if released else None
    engine.set_release(rel)
    for form in FORMS:
        for weighted in (False, True):
            name = _engine_name(form, weighted)
            ww = w if weighted else None
            res = run_search(engine, chains=4096, rounds=24, seed=11, reduced=True, use_dist=False,
                             exchange_every=8, resample_every=4, objective=name, t_start=0.05, t_end=0.01)
            assert sorted(res.prio.tolist()) == list(range(J))
            ref, _ = ST.c_evaluate(tmin, res.opt[None], res.prio[None], f, form, d, ww, rel, True, nodes)
            assert float(ref[0]) == res.makespan
            layouts = set()
            for no_fused in (False, True):
                engine.search_init(2048, seed=3, reduced=True, t_start=0.01, t_end=1e-4, total_rounds=40,
                                   objective=name, _no_fused=no_fused)

                def check(what):
                    assert engine.search_validate() == 0, what
                    opt, prio, score, layout = engine.debug_search_population()
                    want, _ = ST.c_evaluate(tmin, opt, prio, f, form, d, ww, rel, True, nodes)
                    assert score.tobytes() == want.tobytes(), what
                    return layout
                check("init")
                engine.search_seed_lpt()
                check("seeds")
                for n in (1, 3, 16, 17):
                    engine.search_round(n)
                    layouts.add(check("rounds %d, no_fused %s" % (n, no_fused)))
            assert layouts == {0, 2}


def test_completion_seeds_are_the_completion_search_seeds(scen_engine):
    """With every due date +0 the tardiness scenario forms plant the completion search's SPT / WSPT seeds: at K = 1,
    f = 1 the seeded population equals the "completion" / "weighted_completion" one row for row."""
    engine = scen_engine
    J = 64
    T, valid = R.synth_table(J, 3, 8, seed=31)
    engine.set_table(T)
    engine.set_scenarios(np.ones((1, J), np.float32))
    engine.set_due(np.zeros(J, np.float32))
    engine.set_weights(np.random.default_rng(32).uniform(0.5, 3.0, size=J).astype(np.float32))
    for weighted in (False, True):
        rows = []
        for name in (("weighted_" if weighted else "") + "completion",
                     _engine_name("mean_tardiness", weighted), _engine_name("worst_tardiness", weighted)):
            engine.search_init(1024, seed=3, reduced=True, t_start=0.01, t_end=1e-4, total_rounds=4, objective=name,
                               _no_fused=True)
            engine.search_seed_lpt()
            opt, prio, score, _ = engine.debug_search_population()
            rows.append((opt.tobytes(), prio.tobytes(), score.tobytes()))
        assert rows[0] == rows[1] == rows[2], weighted


def _cases():
    with open(os.path.join(HERE, "golden", "scenario_tardiness_cases.json")) as f:
        return json.load(f)["cases"]


def _plan(tasks, out):
    sta, tga, bss, bna, boa, mk = out
    tuples = [[(g, s.runtime) for g, s in t.strategies.items()] for t in tasks]
    assert R.milp_constraints_hold(tuples, sta, tga, bss, bna, boa, mk) == []
    plan = R.plan_from_arrays(tuples, sta, tga, bss, bna)
    for n in sorted({p[5] for p in plan}):
        on = [p for p in plan if p[5] == n]
        ok, ov, _ = R.check_plan([p[0] for p in on], [p[1] for p in on], [p[2] for p in on], [p[3] for p in on])
        assert ok and ov == 0, n


def _kw(rec, obj):
    kw = {"objective": obj, "release": rec["release"], "nodes": rec["nodes"], "weights": rec["weights"]}
    if obj.endswith("tardiness"):
        kw["due"] = rec["due"]
    return kw


def test_solve_reaches_the_exhaustive_optimum():
    """Every fixture instance under all four objectives: solve() returns a plan that passes check_plan and the MILP's
    constraints on the nominal table, whose fp32 device score is the fixture's fp32 exhaustive optimum; last_stats'
    float64 totals are consistent; solve_table on the same table reaches the same score.  Scenarios go in as a
    mapping for solve() and as a sequence for solve_table."""
    from saturn_b200 import solve_table
    from saturn_b200 import solver as S
    for i, rec in enumerate(_cases()):
        tuples = rec["gpu_time_tuples"]
        tasks = tasks_from_tuples(tuples)
        J = len(tasks)
        fT = np.asarray(rec["factors"], dtype=np.float64).T          # [J][K]
        K = fT.shape[1]
        for obj in ST.OBJECTIVES:
            kw = _kw(rec, obj)
            out = S.solve(tasks, None, chains=4096, rounds=60, seed=i,
                          scenarios={t: list(fT[j]) for j, t in enumerate(tasks)}, **kw)
            _plan(tasks, out)
            st = dict(S.last_stats)
            assert st["device_makespan"] == rec[obj + "_f32"]["score"], (rec["name"], obj)
            what = obj.split("_")[1]
            assert len(st["scenario_" + what]) == K and len(st["scenario_makespans"]) == K
            assert st["worst_" + what] == max(st["scenario_" + what])
            assert st["mean_" + what] == pytest.approx(sum(st["scenario_" + what]) / K)
            assert out[5] == pytest.approx(st["makespan"])
            T = np.full((J, 1, 8), np.inf, np.float32)
            for j, tup in enumerate(tuples):
                for g, rt in tup:
                    T[j, 0, int(g) - 1] = rt
            solve_table(T, np.isfinite(T), chains=4096, rounds=60, seed=i, scenarios=fT, **kw)
            assert S.last_stats["device_makespan"] == rec[obj + "_f32"]["score"], (rec["name"], obj)


def test_last_stats_is_a_float64_rescore():
    """On a 64-task set with log-normal factors, last_stats' per-scenario totals are the float64 list schedule of the
    plan's options and order on f * rt (integer starts), within fp32 rounding of the device's score."""
    from saturn_b200 import solver as S
    from saturn_b200.solver import strategies_from_table
    from saturn_b200.synth import synth_table
    J, K = 64, 6
    T, valid = synth_table(J, 4, 8, seed=12)
    st = strategies_from_table(T, valid)
    tasks = [DuckTask("t%d" % j, st[j]) for j in range(J)]
    rng = np.random.default_rng(13)
    fT = rng.lognormal(0.0, 0.3, size=(J, K))
    w = rng.integers(1, 5, size=J).astype(float)
    horizon = float(sum(min(s.runtime for s in t.strategies.values()) for t in tasks)) / 8
    due = np.round(rng.uniform(0.0, horizon, size=J))
    for obj in ST.OBJECTIVES:
        kw = {"due": due} if obj.endswith("tardiness") else {}
        S.solve(tasks, None, chains=8192, rounds=60, seed=2, objective=obj, scenarios=fT, weights=w, **kw)
        s = S.last_stats
        what = obj.split("_")[1]
        vals = s["scenario_" + what]
        score = max(vals) if obj.startswith("worst") else sum(vals)
        assert score == pytest.approx(s["device_makespan"], rel=1e-5, abs=1e-3)
        assert s["worst_" + what] == max(vals)
        assert s["mean_" + what] == pytest.approx(sum(vals) / K, rel=1e-12)


def test_orchestrate_runs_in_simulated_time():
    """orchestrate() with scenarios and due-date mappings keyed by Task runs every task to completion."""
    from saturn_b200 import orchestrate
    rng = np.random.default_rng(9)
    tuples = [[(g, float(rng.uniform(800, 5000)) / g ** 0.8) for g in (1, 2, 4, 8)] for _ in range(8)]
    for obj in ("mean_tardiness", "worst_completion"):
        tasks = tasks_from_tuples(tuples)
        for t in tasks:
            t.total_batches = 200
        kw = {"chains": 4096, "rounds": 25, "objective": obj,
              "scenarios": {t: [1.0, 1.0 + 0.1 * i, 0.8] for i, t in enumerate(tasks)}}
        if obj == "mean_tardiness":
            kw["due"] = {t: 2000.0 + 500.0 * i for i, t in enumerate(tasks)}
        orchestrate(tasks, interval=1000, solver_kwargs=kw, max_intervals=50)
        assert all(t.total_batches == 0 for t in tasks)


def test_multiple_devices_give_a_valid_plan():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from saturn_b200 import solver as S
    rec = _cases()[2]
    tasks = tasks_from_tuples(rec["gpu_time_tuples"])
    for obj in ("worst_tardiness", "mean_completion"):
        kw = _kw(rec, obj)
        out = S.solve(tasks, None, chains=2048, rounds=40, seed=1, devices=2,
                      scenarios=np.asarray(rec["factors"]).T, **kw)
        _plan(tasks, out)
        assert S.last_stats["devices"] == 2
        assert S.last_stats["device_makespan"] == rec[obj + "_f32"]["score"]
