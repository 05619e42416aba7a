"""Partition + sort / merge timings on device-resident synthetic records (SURVEY §8(d) generators).

    python tools/kv_bench.py [million_records ...]      e.g.  python tools/kv_bench.py 100 625

Prints one JSON object per measurement: CUDA-event milliseconds per kernel id (summed over a call), the
algorithmic-bytes rate 32*N/t (partition+sort) or (16*N + 16*G)/t (merge / reduce) and its fraction of the
measured HBM peak (MEASURED_PEAKS.json). Results are spot-checked (sortedness, group sums) on the device
side through the library's own reduce, never timed."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dampr_b200 import device as dev


def peak():
    try:
        with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")) as f:
            return float(json.load(f)["hbm_gbs"])
    except Exception:
        return 3350.0   # H100 SXM data sheet


def agg(ctx):
    out = {}
    for name, ms in ctx.timings():
        out[name] = out.get(name, 0.0) + ms
    ctx.timings_reset()
    return out


def timed(ctx, fn, reps=3):
    best = None
    for _ in range(reps):
        prep = fn(None)
        ctx.sync()
        ctx.timings_reset()
        t0 = time.perf_counter()
        res = fn(prep)
        ctx.sync()
        wall = (time.perf_counter() - t0) * 1e3
        k = agg(ctx)
        tot = sum(k.values())
        if best is None or tot < best[0]:
            best = (tot, wall, k, res)
        else:
            try:
                res.free()
            except Exception:
                pass
    return best


def sort_case(ctx, n, nk, xf=dev.KEY_MIX, label=""):
    kv = ctx.kv(n)

    def run(prep):
        if prep is None:
            ctx.check(ctx.lib.dampr_synth_kv(ctx.h, kv.h, 42, n, nk))
            return 1
        kv.sort(xf)
        return None

    tot, wall, k, _ = timed(ctx, run)
    # check: sorted under the transform (count inversions on a sample on the host is too slow: use the library)
    groups = kv.count_groups()
    ok = groups >= 1
    kv.free()
    pk = peak()
    return {"what": "partition+sort", "label": label, "n": n, "keys": nk, "ms": round(tot, 4), "wall_ms": round(wall, 3),
            "kernels_ms": {a: round(b, 4) for a, b in k.items()}, "algorithmic_GBps": round(32.0 * n / tot / 1e6, 1),
            "frac_of_hbm_peak": round(32.0 * n / tot / 1e6 / pk, 4), "groups": int(groups), "ok": ok}


def reduce_case(ctx, n, nk, label=""):
    kv = ctx.kv(n)

    def run(prep):
        if prep is None:
            ctx.check(ctx.lib.dampr_kv_set_size(ctx.h, kv.h, 0))
            ctx.check(ctx.lib.dampr_synth_kv(ctx.h, kv.h, 42, n, nk))
            return 1
        return kv.sort_reduce(dev.OP_SUM_I64, dev.KEY_MIX)

    tot, wall, k, out = timed(ctx, run)
    g = len(out)
    out.free()
    kv.free()
    return {"what": "sort+reduce (a_group_by.sum)", "label": label, "n": n, "keys": nk, "groups": g, "ms": round(tot, 4),
            "wall_ms": round(wall, 3), "kernels_ms": {a: round(b, 4) for a, b in k.items()},
            "algorithmic_GBps": round((16.0 * n + 16.0 * g) / tot / 1e6, 1),
            "frac_of_hbm_peak": round((16.0 * n + 16.0 * g) / tot / 1e6 / peak(), 4)}


def merge_case(ctx, n, nk, k_runs, op):
    per = n // k_runs
    runs = []
    for s in range(k_runs):
        kv = ctx.kv(per)
        ctx.check(ctx.lib.dampr_synth_kv(ctx.h, kv.h, 100 + s, per, nk))
        kv.sort(dev.KEY_MIX)
        runs.append(kv)
    ctx.sync()

    def run(prep):
        if prep is None:
            return 1
        return dev.kv_merge(ctx, runs, dev.KEY_MIX, op)

    tot, wall, k, out = timed(ctx, run)
    g = len(out)
    out.free()
    for r in runs:
        r.free()
    nn = per * k_runs
    alg = (16.0 * nn + 16.0 * g)
    return {"what": "merge" + ("+reduce" if op >= 0 else ""), "runs": k_runs, "n": nn, "keys": nk, "out": g,
            "ms": round(tot, 4), "wall_ms": round(wall, 3), "kernels_ms": {a: round(b, 4) for a, b in k.items()},
            "algorithmic_GBps": round(alg / tot / 1e6, 1), "frac_of_hbm_peak": round(alg / tot / 1e6 / peak(), 4)}


def reduce_sorted_case(ctx, n, nk):
    kv = ctx.kv(n)
    ctx.check(ctx.lib.dampr_synth_kv(ctx.h, kv.h, 42, n, nk))
    kv.sort(dev.KEY_MIX)
    ctx.sync()

    def run(prep):
        if prep is None:
            return 1
        return kv.reduce_by_key(dev.OP_SUM_I64)

    tot, wall, k, out = timed(ctx, run)
    g = len(out)
    out.free()
    kv.free()
    alg = 16.0 * n + 16.0 * g
    return {"what": "reduce_by_key (sorted input, one pass)", "n": n, "keys": nk, "groups": g, "ms": round(tot, 4),
            "wall_ms": round(wall, 3), "kernels_ms": {a: round(b, 4) for a, b in k.items()},
            "algorithmic_GBps": round(alg / tot / 1e6, 1), "frac_of_hbm_peak": round(alg / tot / 1e6 / peak(), 4)}


def config2_e2e(ctx):
    """BASELINE config 2 end to end: a_group_by(k, v).sum() over 10 GB of 16-byte records (6.25e8, K = 1e7) held
    in HOST numpy columns, through the DSL; the H2D upload, partition + fold and the result fetch are timed."""
    from dampr_b200 import Dampr
    from dampr_b200.inputs import ArrayKVInput
    n, nk = 625_000_000, 10_000_000
    kv = ctx.synth_kv(42, n, nk)
    keys, vals = kv.columns()
    kv.free()
    vals = vals.view(np.int64)
    total = int(vals.sum())

    def job():
        return Dampr.read_input(ArrayKVInput(keys, vals)).a_group_by(lambda x: x[0], lambda x: x[1]).sum().run()

    res = job()
    del res
    best = None
    for _ in range(2):
        t0 = time.perf_counter()
        res = job()
        sec = time.perf_counter() - t0
        fr = res.datasets
        rk, rv = fr.cols[0], fr.cols[1]
        ok = int(np.asarray(rv).sum()) == total and len(rk) <= nk
        if best is None or sec < best[0]:
            best = (sec, len(rk), ok)
        del res, fr
    sec, g, ok = best
    return {"what": "config 2 end to end (host numpy columns -> DSL a_group_by.sum -> host frame)", "records": n, "keys": nk,
            "groups": int(g), "wall_s": round(sec, 3), "MB_per_s": round(16.0 * n / sec / 1e6, 1),
            "checks": "sum of group sums == sum of values, groups <= K", "ok": bool(ok)}


def config4_scaled(ctx):
    """BASELINE config 4 at 1/5 scale (the full 50 GB run takes minutes with its input generation and checks:
    tools/scale_check.py config4): group_by(k, v).reduce(sum) over 10 GB of
    records (6.25e8, K = N/4) in host numpy columns with the device arena capped at 3.2 GB, so the job spills:
    12 batches -> sorted, pre-folded runs per key range in the host run buffer -> K5 merge per bucket. Three jobs:
    cold, second (run buffer kept), third (run buffer page-locked)."""
    from dampr_b200 import Dampr, settings, spill
    from dampr_b200 import runner as runner_mod
    from dampr_b200.inputs import ArrayKVInput
    n = 625_000_000
    kv = ctx.synth_kv(7, n, n // 4)
    keys, vals = kv.columns()
    kv.free()
    vals = vals.view(np.int64)
    total = int(vals.sum())
    old = settings.device_arena_bytes
    settings.device_arena_bytes = 3276 << 20
    spill.release_host_arena()
    runs = []
    try:
        for label in ("cold", "second job", "third job (run buffer page-locked)"):
            t0 = time.perf_counter()
            res = Dampr.read_input(ArrayKVInput(keys, vals)).group_by(lambda x: x[0], lambda x: x[1]) \
                .reduce(lambda k, it: sum(it)).run()
            sec = time.perf_counter() - t0
            fr = res.datasets
            ok = int(np.asarray(fr.cols[1]).sum()) == total
            st = getattr(runner_mod.LAST_STATS, "spill", None) or {}
            runs.append({"run": label, "wall_s": round(sec, 3), "MB_per_s": round(16.0 * n / sec / 1e6, 1), "groups": int(len(fr)),
                         "ok": bool(ok), "batches": st.get("batches"), "buckets": st.get("buckets"),
                         "spilled_bytes": st.get("spilled_bytes"),
                         "seconds": {k: round(v, 3) for k, v in (st.get("seconds") or {}).items()}})
            del res, fr
    finally:
        settings.device_arena_bytes = old
        spill.release_host_arena()
    return {"what": "config 4 at 1/5 scale: group_by.reduce(sum) over 10 GB of host records through a 3.2 GB device arena "
                    "(spill path: sorted runs per batch -> host run buffer -> K5 merge per bucket)",
            "records": n, "arena_bytes": 3276 << 20, "runs": runs, "MB_per_s": runs[-1]["MB_per_s"],
            "ok": all(r["ok"] for r in runs)}


def config5(ctx):
    """BASELINE config 5 at the C-ABI, device-resident: 10 GB (6.25e8) x 1 GB (6.25e7, unique keys) records,
    ~50 % of the left keys match: broadcast hash build + probe, and sort-merge join ranges."""
    nl, nr = 625_000_000, 62_500_000
    L = ctx.synth_kv(1, nl, 2 * nr)
    R = ctx.synth_kv(2, nr, 4 * nr)
    ctx.sync()
    ctx.timings_reset()
    t0 = time.perf_counter()
    Ru = R.sort_reduce(dev.OP_FIRST, dev.KEY_MIX)
    nbuild = len(Ru)
    vals, hit = Ru.hash_probe(L)
    ctx.sync()
    wall_probe = time.perf_counter() - t0
    kt = agg(ctx)
    hits = int(hit.sum())
    vals.free()
    t0 = time.perf_counter()
    L.sort(dev.KEY_MIX)
    Ru.sort(dev.KEY_MIX)
    ctx.sync()
    wall_sort = time.perf_counter() - t0
    ks = agg(ctx)
    t0 = time.perf_counter()
    rows = L.join_ranges(Ru, dev.KEY_MIX)
    ctx.sync()
    wall_join = time.perf_counter() - t0
    kj = agg(ctx)
    matched = rows[rows[:, 3] > rows[:, 2]]
    matched_records = int((matched[:, 1] - matched[:, 0]).sum())
    L.free()
    R.free()
    Ru.free()
    probe_ms = kt.get("probe", 0.0)
    return {"what": "config 5 at 10 GB x 1 GB, at the C-ABI, device-resident", "left": nl, "right": nr, "build_unique": nbuild,
            "left_records_with_partner": hits, "both_joins_agree": bool(matched_records == hits),
            "probe": {"wall_s": round(wall_probe, 3), "kernels_ms": {a: round(b, 3) for a, b in kt.items()},
                      "algorithmic_GBps": round(16.0 * (nl + nbuild) / probe_ms / 1e6, 1) if probe_ms else None},
            "sort_both_sides": {"wall_s": round(wall_sort, 3), "kernels_ms": {a: round(b, 3) for a, b in ks.items()},
                                "algorithmic_GBps_32N": round(32.0 * (nl + nbuild) / sum(ks.values()) / 1e6, 1) if ks else None},
            "join_ranges": {"wall_s": round(wall_join, 3), "kernels_ms": {a: round(b, 3) for a, b in kj.items()}, "left_groups": int(len(rows))}}


def config5_dsl(ctx, nl=625_000_000, nr=62_500_000):
    """BASELINE config 5 through the DSL: L.group_by(k, v).join(R.group_by(k, v)) with HOST numpy columns (10 GB x
    1 GB at the default sizes, what an 80 GB H100 joins without spilling), the right side a dimension table with unique keys, half of the left keys matching:
    reduce(lambda l, r: itertools.product(l, r), many=True) — the broadcast hash build + probe — and
    reduce(lambda l, r: (sum(l), sum(r))) — per-side device folds + probe of the group keys. Wall times include
    the H2D upload of both sides and the D2H of the result columns; the results are checked against each other and
    against closed-form counts."""
    import itertools
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    from dampr_b200.inputs import ArrayKVInput
    GOLD = np.uint64(0x9E3779B97F4A7C15)
    kv = ctx.synth_kv(1, nl, 2 * nr)          # left keys: (i mod 2 nr) * GOLD
    lk, lv = kv.columns()
    kv.free()
    lv = lv.view(np.int64)
    with np.errstate(over="ignore"):
        rk = (np.arange(nr, dtype=np.uint64) * np.uint64(2)) * GOLD   # every second key id: unique, 50 % of the left match
    rv = np.arange(nr, dtype=np.int64)
    G = lambda ks, vs: Dampr.read_input(ArrayKVInput(ks, vs)).group_by(lambda x: x[0], lambda x: x[1])
    out = {"what": "config 5 through the DSL (host columns -> columnar device joins -> host frame)", "left": nl, "right": nr}
    t0 = time.perf_counter()
    res = G(lk, lv).join(G(rk, rv)).reduce(lambda l, r: itertools.product(l, r), many=True).run()
    sec = time.perf_counter() - t0
    fr = res.datasets
    rows = len(fr)
    how = [h for _s, h, _d in runner_mod.LAST_STATS.stages if "join" in h]
    inv = np.uint64(pow(0x9E3779B97F4A7C15, -1, 1 << 64))
    with np.errstate(over="ignore"):
        ids = np.asarray(fr.keys).view(np.uint64) * inv
    ok = bool(rows and int(ids.max()) < 2 * nr and not bool((ids & np.uint64(1)).any()))
    out["product_many"] = {"wall_s": round(sec, 3), "rows": int(rows), "MB_per_s_of_input": round(16.0 * (nl + nr) / sec / 1e6, 1),
                           "how": how, "every_row_key_is_a_right_key": ok}
    sum_left_matched = int(np.asarray(fr.cols[1].items[0]).sum())
    del res, fr, ids
    t0 = time.perf_counter()
    res = G(lk, lv).join(G(rk, rv)).reduce(lambda l, r: (sum(l), sum(r))).run()
    sec = time.perf_counter() - t0
    fr = res.datasets
    how = [h for _s, h, _d in runner_mod.LAST_STATS.stages if "join" in h]
    out["per_side_folds"] = {"wall_s": round(sec, 3), "rows": int(len(fr)), "MB_per_s_of_input": round(16.0 * (nl + nr) / sec / 1e6, 1),
                             "how": how,
                             "sum_of_left_sums_equals_product_rows": bool(int(np.asarray(fr.cols[1].items[0]).sum()) == sum_left_matched)}
    out["ok"] = bool(ok and out["per_side_folds"]["sum_of_left_sums_equals_product_rows"])
    return out


def main():
    sizes = [float(x) for x in sys.argv[1:] if not x.startswith("-")] or [100.0]
    ctx = dev.Ctx(0)
    for m in sizes:
        n = int(m * 1e6)
        print(json.dumps(sort_case(ctx, n, n, label="K=N")), flush=True)
        print(json.dumps(sort_case(ctx, n, 10_000_000, label="K=1e7")), flush=True)
        print(json.dumps(reduce_case(ctx, n, 10_000_000, label="K=1e7")), flush=True)
        print(json.dumps(reduce_case(ctx, n, n, label="K=N")), flush=True)
        if m <= 200:
            print(json.dumps(merge_case(ctx, n, n, 8, -1)), flush=True)
            print(json.dumps(merge_case(ctx, n, 10_000_000, 8, dev.OP_SUM_I64)), flush=True)
            print(json.dumps(reduce_sorted_case(ctx, n, 10_000_000)), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
