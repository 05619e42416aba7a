"""The engine against the REAL reference (Refefer/Dampr) at the sizes and keys where the kv kernels change regime:
the 4 096-record leaf, partition and offset tiles (4 095 / 4 096 / 4 097 records), 2^16 + 1 records, and 300 000
and 1 200 000 records. (The tile scans' second pass, beyond 1 024 tiles of 4 096 records, is tested through the C ABI
in tests/test_gpu_join_probe.py.) Key pools: distinct keys,
n/3, 7 and 1 key, Zipf(1.1), the int64 extremes, ints next to +-2^53 mixed with floats (the FLOAT / HASH boundary of
keycodec._classify), ints >= 2^63, floats with infinities and subnormals, strings sharing a long prefix and non-ASCII
strings, tuples, keys whose mix64 all land in one sort bucket and one probe slot, and equal keys of different types
(0 / 0.0 / -0.0 / False). Values near 2^62 make int sums leave int64, where the fold must hand over to Python ints.

Inputs are generated inside the reference's interpreter and here by the same integer code (GEN: splitmix64), so no
item list travels on a command line. Per pipeline the reference's result is recorded as its length and the sha256
of its sorted reprs (tests/golden/differential_seams.json.gz): outputs are compared as multisets. Pipelines whose
output key object depends on the reference's worker scheduling (equal keys of different types) run on one input
partition. The stand-in for the device (tests/fake_device.py) runs the groups up to 65 537 records; the larger ones
run on the device only. Every case states the path its keyed stage takes, and on the device that kernels ran."""
import hashlib
import json
import os
import sys

import pytest

from test_differential_reference import REF, Engine, ReferenceReplay

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "differential_seams.json.gz")
subprocess = ReferenceReplay(GOLDEN)

GEN = r'''
import bisect
M64 = (1 << 64) - 1


def splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def unmix64(t):
    """the inverse of the device's mix64 (csrc/common.cuh)"""
    t ^= (t >> 31) ^ (t >> 62)
    t = (t * 0x319642B2D24D8EC3) & M64
    t ^= (t >> 27) ^ (t >> 54)
    t = (t * 0x96DE1B173F119089) & M64
    t ^= (t >> 30) ^ (t >> 60)
    return t


# Zipf(1.1) over 50 000 keys; weights quantised coarsely enough that the last bit of pow() cannot move them
ZIPF = []
_acc = 0
for _k in range(1, 50001):
    _acc += int(2.0 ** 30 * _k ** -1.1) + 1
    ZIPF.append(_acc)
EXT = [-2 ** 63, 2 ** 63 - 1, -2 ** 63 + 1, 2 ** 63 - 2, 0, -1, 1]
NEAR53 = [2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, 2 ** 53 + 2, -2 ** 53 - 1, -2 ** 53, -2 ** 53 + 1, float(2 ** 53),
          float(2 ** 53 + 2), -float(2 ** 53), 0.5, 2.0 ** 54]
FLOATS = [float("inf"), float("-inf"), 5e-324, -5e-324, 2.2250738585072014e-308, 1e-310, -1e-310]
EQREPR = [0, 0.0, -0.0, False, 1, 1.0, True, 2, 2.0]
# mix64(key) = 0x5A5 in the top 12 bits (one sort bucket) and 0xFFFFD in the low 20 (slot cap - 3 of every probe
# table up to 2^20 slots)
UNMIX = [unmix64((0x5A5 << 52) | (j << 20) | 0xFFFFD) for j in range(4096)]


def key_of(pool, i, r, n):
    if pool == "distinct":
        k = (i * 0x9E3779B97F4A7C15) & M64
        return k - (1 << 64) if k >> 63 else k
    if pool == "third":
        return r % max(1, n // 3)
    if pool == "seven":
        return r % 7 - 3
    if pool == "one":
        return 17
    if pool == "zipf":
        return bisect.bisect_right(ZIPF, r % ZIPF[-1])
    if pool == "i64ext":
        return EXT[(r >> 1) % len(EXT)] if r & 1 else (r >> 1) % 1000 - 500
    if pool == "near53":
        return NEAR53[r % len(NEAR53)]
    if pool == "big":
        return 2 ** 63 + (r >> 1) % 1000 if r & 1 else 2 ** 64 + (r >> 1) % 50 if r & 2 else 2 ** 70 + r % 3
    if pool == "floats":
        return FLOATS[(r >> 1) % len(FLOATS)] if r & 1 else (r >> 1) % 500 / 8.0
    if pool == "prefix":
        c = r % 3
        return "shared-prefix-key/%d" % (r % 300) if c == 0 else "ключ-%d" % (r % 50) if c == 1 \
            else "鍵%dé" % (r % 40)
    if pool == "tuples":
        return (r % 13, "k%d" % (r % 5))
    if pool == "unmix":
        return UNMIX[r % len(UNMIX)]
    if pool == "eqrepr":
        return EQREPR[r % len(EQREPR)]
    raise ValueError(pool)


def val_of(vals, r):
    if vals == "small":
        return r % 2001 - 1000
    if vals == "huge":
        return -(1 << 62) - r % 1000 if r % 4 == 0 else (1 << 62) + r % 1000
    if vals == "ties":
        return r % 10
    raise ValueError(vals)


def make_items(pool, vals, n, seed):
    out = []
    for i in range(n):
        r = splitmix64(seed * 1000003 + i)
        out.append((key_of(pool, i, r, n), val_of(vals, splitmix64(r ^ 0x5851F42D4C957F2D))))
    return out


def make_other(kind, items):
    """the right side of a join / the build side of a probe"""
    n = len(items)
    if kind == "subset":
        return [(k + 1 if type(k) is int else k, v) for k, v in items[n // 4::3]]
    if kind == "empty":
        return []
    if kind == "hot":
        return [(items[0][0], v) for _k, v in items[::5]] if items else []
    if kind == "unmix":
        return [(k, j) for j, k in enumerate(UNMIX[::2])]
    return []
'''

DRIVER = GEN + r'''
import sys, json, hashlib
sys.path.insert(0, sys.argv[1])
from dampr import Dampr
res = []
for c in json.loads(sys.argv[2]):
    items = make_items(c["pool"], c["vals"], c["n"], c["seed"])
    other = make_other(c["other"], items)
    r = list(eval(c["src"]).run())
    res.append([len(r), hashlib.sha256("\n".join(sorted(repr(x) for x in r)).encode()).hexdigest()])
print(json.dumps(res))
'''

G = {}
exec(GEN, G)

A = "Dampr.memory(items, partitions=%d)"
B = "Dampr.memory(other, partitions=2)"
# op -> (pipeline tail, the path its keyed stage takes)
OPS = {
    "sum": (".fold_by(lambda x: x[0], lambda a, b: a + b, lambda x: x[1])", "host-map + device shuffle/combine"),
    "min": (".fold_by(lambda x: x[0], min, lambda x: x[1])", "host-map + device shuffle/combine"),
    "max": (".fold_by(lambda x: x[0], max, lambda x: x[1])", "host-map + device shuffle/combine"),
    "count": (".count(lambda x: x[0])", "host-map + device shuffle/combine"),
    "agsum": (".a_group_by(lambda x: x[0], lambda x: x[1]).sum()", "host-map + device shuffle/combine"),
    "mean": (".mean(lambda x: x[0], lambda x: x[1])", "host-map + device shuffle/combine"),
    "glen": (".group_by(lambda x: x[0], lambda x: x[1]).reduce(lambda k, it: len(list(it)))",
             "host-map + device shuffle"),
    "sort": (".sort_by(lambda x: x[1])", "host-map + device shuffle"),
    "len": (".len()", "host-map + device shuffle"),
    "unique": (".group_by(lambda x: x[0], lambda x: x[1]).unique()", "host-map + device shuffle"),
    "topk": (".topk(5, lambda x: x[1])", None),
    "join": (".group_by(lambda x: x[0], lambda x: x[1]).join(" + B + ".group_by(lambda x: x[0], lambda x: x[1]))"
             ".reduce(lambda l, r: (sum(l), sum(r)))", "device join ranges + host aggregate"),
    "left": (".group_by(lambda x: x[0], lambda x: x[1]).join(" + B + ".group_by(lambda x: x[0], lambda x: x[1]))"
             ".left_reduce(lambda l, r: (sum(l), len(list(r))))", "device join ranges + host aggregate"),
}


def case(pool, vals, n, op, partitions=3, other="", seed=1):
    tail, how = OPS[op]
    if op in ("unique", "topk") or pool in ("near53", "eqrepr"):
        partitions = 1
    return {"pool": pool, "vals": vals, "n": n, "seed": seed, "other": other, "src": A % partitions + tail, "how": how}


def probe_case(n, seed=1):
    """cross_set membership of the unmix pool's keys in a build side of crafted keys. Here both sides are binary
    (key, value) inputs, which take the device's broadcast hash probe."""
    tail = ".map(lambda x: x[0]).cross_set(%s, lambda b, table: (b[0], b[1], b[0] in table), agg=set)"
    return {"pool": "unmix", "vals": "small", "n": n, "seed": seed, "other": "unmix", "src": B + tail % (A % 3),
            "ours": "Dampr.read_input(ArrayKVInput(K2, V2))" + tail % "Dampr.read_input(ArrayKVInput(K, V))",
            "how": "device broadcast hash build+probe"}


def columns(records):
    import numpy as np
    k = np.array([r[0] for r in records], dtype=np.uint64)
    return k, np.array([r[1] for r in records], dtype=np.int64)


SEAMS = [0, 1, 4095, 4096, 4097, 65537]
FOLDS = ["sum", "min", "max", "count", "agsum", "mean", "glen", "sort", "len"]
POOLS = ["distinct", "seven", "one", "zipf", "i64ext", "near53", "big", "floats", "prefix", "tuples", "unmix", "eqrepr"]
GROUPS = {
    # every fold at every tile seam up to 2^16 + 1 records
    "seams": [case("third", "small", n, op) for n in SEAMS for op in FOLDS],
    # every key pool through the folds, group sizes and a join, at 4 097 records
    "pools": [case(pool, "small", 4097, op, seed=7) for pool in POOLS for op in ("sum", "count", "min", "glen")] +
             [case(pool, "small", 4097, "join", other="subset", seed=7) for pool in POOLS
              if pool not in ("near53", "eqrepr")],
    # sums that leave int64; unique and topk (ties at the cut); joins against shifted, empty and one-key sides
    "values": [case(pool, "huge", n, op, seed=3) for pool in ("seven", "distinct") for n in (4097, 65537)
               for op in ("sum", "agsum", "mean")] +
              [case("third", "small", n, "unique") for n in (4095, 4097, 65537)] +
              [case("zipf", "ties", n, "topk") for n in (4097, 65537)],
    "joins": [case("third", "small", n, op, other=o, seed=5) for n in (1, 4096, 4097, 65537) for op in ("join", "left")
              for o in ("subset", "empty", "hot")],
    "probe": [probe_case(n) for n in (0, 1, 4097, 65537)],
    # device only: 300 000 records (74 tiles of 4 096) and 1 200 000 records (293 tiles)
    "large": [case("third", "small", 300000, op) for op in FOLDS] +
             [case("zipf", "small", 300000, op, seed=9) for op in ("sum", "glen", "join")] +
             [case("third", "small", 300000, op, other="subset") for op in ("join", "left")] +
             [case("seven", "huge", 300000, "sum"), case("third", "small", 300000, "unique"), probe_case(300000)],
    "million": [case("third", "small", 1200000, op, seed=11) for op in ("sum", "count", "glen", "sort")] +
               [case("third", "small", 1200000, "join", other="subset", seed=11), probe_case(1200000, seed=11)],
}
DEVICE_ONLY = ("large", "million")


def digest(result):
    rs = sorted(repr(x) for x in result)
    return [len(rs), hashlib.sha256("\n".join(rs).encode()).hexdigest()]


def reference(cases):
    env = dict(os.environ)
    env.pop("PYTHONPATH", None)
    spec = [{k: c[k] for k in ("pool", "vals", "n", "seed", "other", "src")} for c in cases]
    p = subprocess.run([sys.executable, "-c", DRIVER, REF, json.dumps(spec)], capture_output=True, text=True, env=env,
                       cwd="/tmp", timeout=1200)
    assert p.returncode == 0, p.stderr[-2000:]
    return json.loads(p.stdout.strip().split("\n")[-1])


PARAMS = [pytest.param("device", g, marks=pytest.mark.gpu, id="device-" + g) for g in GROUPS] + \
         [pytest.param("fake", g, id="fake-" + g) for g in GROUPS if g not in DEVICE_ONLY]


@pytest.mark.parametrize("kind,group", PARAMS)
def test_seams_agree_with_the_reference(kind, group, monkeypatch):
    from dampr_b200 import Dampr, plan
    cases = GROUPS[group]
    ref = reference(cases)
    assert len(ref) == len(cases)
    engine = Engine(kind, monkeypatch)
    try:
        for c, exp in zip(cases, ref):
            items = G["make_items"](c["pool"], c["vals"], c["n"], c["seed"])
            other = G["make_other"](c["other"], items)
            engine.use()
            ns = {"Dampr": Dampr, "items": items, "other": other}
            if "ours" in c:
                from dampr_b200.inputs import ArrayKVInput
                (K, V), (K2, V2) = columns(items), columns(other)
                ns.update(ArrayKVInput=ArrayKVInput, K=K, V=V, K2=K2, V2=V2)
            got = digest(eval(c.get("ours", c["src"]), ns).run())
            hows = engine.hows()
            assert got == exp, (c["pool"], c["vals"], c["n"], c["src"])
            if c["how"] is not None and c["n"]:
                assert c["how"] in hows, (c["src"], hows)
        engine.ran_on_device()
    finally:
        if engine.device:
            plan.release_buffers()


def test_every_group_has_a_recording():
    """The recordings of all groups, the device-only ones included (with DAMPR_REFERENCE set this records them). The
    reference shows one of several equal keys (0 / 0.0 / False); on one input partition it is always the same one,
    which a second recording of those pipelines confirms."""
    for group, cases in GROUPS.items():
        ref = reference(cases)
        assert len(ref) == len(cases) and all(len(d) == 2 and len(d[1]) == 64 for d in ref), group
    mixed = [c for c in GROUPS["pools"] if c["pool"] in ("eqrepr", "near53")]
    assert mixed and all("partitions=1" in c["src"] for c in mixed)
    if REF:
        import subprocess as sp
        env = dict(os.environ)
        env.pop("PYTHONPATH", None)
        spec = [{k: c[k] for k in ("pool", "vals", "n", "seed", "other", "src")} for c in mixed]
        p = sp.run([sys.executable, "-c", DRIVER, REF, json.dumps(spec)], capture_output=True, text=True, env=env,
                   cwd="/tmp", timeout=600)
        assert p.returncode == 0, p.stderr[-2000:]
        first = reference(GROUPS["pools"])
        assert json.loads(p.stdout.strip().split("\n")[-1]) == [d for c, d in zip(GROUPS["pools"], first) if c in mixed]
