"""The long-key collision guard of the text and field kernels, on real 64-bit code collisions.

Tokens and field keys too long for an exact code share a 64-bit hashed code with other strings; the pairs in
tests/golden/code_collisions.json do (tests/test_code_collisions.py states the codes in Python). Every kernel
byte-compares the strings behind a shared code and sets DAMPR_TF_COLLISION on a mismatch, and the planner then runs
the stage on the host. Here: the kernels give the codes the Python statement gives (so the collision tests cannot pass
vacuously after a change of hash or seed); every build of the tokenise kernels, in every mode, flags a pair wherever
the two strings sit (same line, set() rounds and history, strips, tiles, halo, range cuts, the str.split combiner) and
is otherwise exact; the field fold flags colliding keys in table and record mode; and the DSL pipelines return
Python's answers through the host path."""
import collections
import functools
import logging
import random
import re

import numpy as np
import pytest

import text_contract as tc
from dampr_b200 import device as dev
from fields_standin import write_files
from test_code_collisions import PAIRS, key_code
from test_gpu_text_seams import Scan

pytestmark = pytest.mark.gpu

BUILDS = [(2, 4), (2, 3), (2, 2), (1, 2)]
MODES = (tc.TOK_WS, tc.TOK_NONWORD_LOWER_SET, tc.TOK_NONWORD_LOWER)
NONWORD = (tc.TOK_NONWORD_LOWER_SET, tc.TOK_NONWORD_LOWER)
REFUSE = tc.TF_NONASCII | tc.TF_LONGLINE | tc.TF_TABLEFULL
ALNUM = b"abcdefghijklmnopqrstuvwxyz0123456789"
RX = re.compile(r"[^\w]+")


@pytest.fixture(params=BUILDS, ids=["v2-4cta", "v2-3cta", "v2-2cta", "v1"])
def build(request):
    dev.set_option("text_kernel", request.param[0])
    dev.set_option("text_ctas", request.param[1])
    try:
        yield request.param
    finally:
        dev.set_option("text_kernel", 2)
        dev.set_option("text_ctas", 4)


def variant(mode):
    return "raw" if mode == tc.TOK_WS else "sym"


def word(rng, n):
    return bytes(rng.choice(ALNUM) for _ in range(n))


# ---- placements of a pair (a, b) -----------------------------------------------------------------------------------
# each returns the text and the offset of the first line holding b; PLACEMENTS names beside each the modes in which two
# tokens the device counts share a code (case variants only do in the [^\w]+ modes)
def _w(rng, n_filler=20):
    w = tc.Writer(rng)
    for _ in range(n_filler):
        w.filler_line()
    return w


def _fin(w, b_off, n_filler=20):
    for _ in range(n_filler):
        w.filler_line()
    return w.data(), b_off


def p_adjacent(a, b, rng):
    w = _w(rng)
    off = len(w.buf)
    w.line(b"x " + a + b" " + b + b" y")
    return _fin(w, off)


def p_apart(a, b, rng):
    """45 distinct tokens between them: b is in a later 32-token round, found by the set() history"""
    w = _w(rng)
    off = len(w.buf)
    w.line(b" ".join([b"q", a] + [b"w%d" % i for i in range(45)] + [b, b"z"]))
    return _fin(w, off)


def p_second_only(a, b, rng):
    """a on many lines, b only once, as the second of the pair on its line"""
    w = _w(rng)
    for i in range(40):
        w.line(b"k%d " % i + a + b" tail")
        if i == 20:
            off = len(w.buf)
            w.line(b"k " + a + b", " + b)
    return _fin(w, off)


def p_same_strip(a, b, rng):
    w = _w(rng, 3)
    w.line(b"one " + a)
    w.filler_line()
    off = len(w.buf)
    w.line(b"two " + b)
    return _fin(w, off)


def p_other_strip(a, b, rng):
    w = _w(rng, 3)
    w.line(b"one " + a)
    w.pad_to(3 * tc.V_STRIP + 300)
    off = len(w.buf)
    w.line(b"two " + b)
    return _fin(w, off)


def p_other_tile(a, b, rng):
    w = _w(rng, 3)
    w.line(b"one " + a)
    w.pad_to(2 * tc.V_OWN + 5000)
    off = len(w.buf)
    w.line(b"two " + b)
    return _fin(w, off)


def p_halo(a, b, rng):
    """b's line starts 40 bytes before a tile seam and b lies past it: the tile before reads b from its halo"""
    w = _w(rng, 3)
    w.line(b"one " + a)
    w.pad_to(2 * tc.V_OWN - 40)
    off = len(w.buf)
    w.line(b" ".join(b"f%d" % i for i in range(20)) + b" " + b)
    assert off < 2 * tc.V_OWN < w.buf.index(b, off)
    return _fin(w, off)


def p_zipf(a, b, rng):
    """a thousands of times (str.split: the shared-memory combiner and its representative), b once at the end"""
    w = _w(rng, 3)
    for i in range(6000):
        w.line(a + b" %s" % word(rng, rng.randint(1, 6)) if i % 3 else a)
    off = len(w.buf)
    w.buf += b + b"\n"
    return w.data(), off


def p_long32(a, b, rng):
    s = word(rng, 30)
    return p_adjacent(a + s, b + s, rng)


def p_long4k(a, b, rng):
    s = word(rng, 4000)
    w = _w(rng, 5)
    w.line(b"x " + a + s)
    off = len(w.buf)
    w.line(b"y " + b + s)      # (one 4 KB token per line: the first-generation kernel's window holds such lines)
    w.line(a + s)
    return _fin(w, off)


def p_mixed_case(a, b, rng):
    ua = bytes(c - 32 if 0x61 <= c <= 0x7A and rng.random() < 0.5 else c for c in a)
    return p_adjacent(ua, b.upper(), rng)


def p_host_line(a, b, rng):
    """b only on a line with a non-ASCII byte: the [^\\w]+ modes hand that line to the host, no flag is needed"""
    w = _w(rng)
    w.line(b"one " + a)
    off = len(w.buf)
    w.line("café ".encode() + b)
    return _fin(w, off)


def p_repeat(a, b, rng):
    """negative control: one long word many times on a line and on others"""
    w = _w(rng)
    off = len(w.buf)
    w.line(b" ".join([a] * 50 + [b"w%d" % i for i in range(40)] + [a]))
    w.line(a + b" " + a)
    return _fin(w, off)


def p_case_variants(a, b, rng):
    """negative control: case variants of one word on one line"""
    w = _w(rng)
    off = len(w.buf)
    w.line(b" ".join([a, a.upper(), a.capitalize()] + [b"w%d" % i for i in range(40)] + [a.swapcase()]))
    return _fin(w, off)


ALL = set(MODES)
PLACEMENTS = {
    "adjacent": (p_adjacent, ALL), "apart_45": (p_apart, ALL), "second_only": (p_second_only, ALL),
    "same_strip": (p_same_strip, ALL), "other_strip": (p_other_strip, ALL), "other_tile": (p_other_tile, ALL),
    "halo": (p_halo, ALL), "zipf": (p_zipf, ALL), "long32": (p_long32, ALL), "long4k": (p_long4k, ALL),
    "mixed_case": (p_mixed_case, set(NONWORD)), "host_line": (p_host_line, {tc.TOK_WS}),
    "repeat": (p_repeat, set()), "case_variants": (p_case_variants, set()),
}


@functools.lru_cache(maxsize=None)
def placed(name, var):
    rng = random.Random(name + var)
    pairs = PAIRS[var]
    a, b, _s, _c = pairs[sorted(PLACEMENTS).index(name) % len(pairs)]
    return PLACEMENTS[name][0](a, b, rng)


def cuts(data, b_off):
    """the contract's ownership splits, and one cut right before b's line"""
    out = dict(tc.cut_sets(len(data)))
    c = b_off // 16 * 16
    if 0 < c < len(data):
        out["before_b"] = [(0, c), (c, len(data))]
    return out


def counted_collides(exp_table, mode):
    """two different tokens of the table the device keeps share a code"""
    toks = [t.encode() for t in exp_table]
    return len({key_code(t, variant(mode)) for t in toks}) < len(toks)


def check(scan, build, mode, cut, ranges, declared):
    """the contract: TF_COLLISION when two counted tokens share a code, an exact table otherwise"""
    kernel, ctas = build
    data = scan.data
    st = scan.count(mode, False, ranges)
    if kernel == 1:
        scan.tab.verify(scan.tb, 0, len(data), mode)
        st = scan.tab.stats()
    flags = st["flags"]
    req, allowed = tc.refusals(data, mode, False, ranges, kernel, ctas)
    where = (build, mode, cut, flags)
    assert flags & req == req, where
    if req & REFUSE:
        return "refused"
    fb = tc.expected_fallback(data, kernel, mode, False)
    exp = tc.expected_table(data, mode, False, fb)
    collides = counted_collides(exp["table"], mode)
    assert collides == (mode in declared), where      # the placement holds what it says it does
    if collides:
        assert flags & tc.TF_COLLISION, where
        return "flagged"
    assert flags & ~allowed == 0, where
    assert sorted(scan.tab.fallback_lines().tolist()) == fb, where
    got = scan.table(mode)
    assert got == exp["table"], (where, sorted(set(got.items()) ^ set(exp["table"].items()))[:10])
    assert (st["lines"], st["folded"]) == (exp["lines"], exp["folded"]), (where, st)
    if mode != tc.TOK_WS:
        assert st["empty"] == exp["empty"], where
    return "exact"


@pytest.mark.parametrize("name", sorted(PLACEMENTS))
def test_tokenise_kernels_flag_colliding_tokens(ctx, build, name):
    outcomes = collections.Counter()
    for var in ("raw", "sym"):
        data, b_off = placed(name, var)
        scan = Scan(ctx, data)
        try:
            for mode in (m for m in MODES if variant(m) == var):
                for cut, ranges in sorted(cuts(data, b_off).items()):
                    outcomes[check(scan, build, mode, cut, ranges, PLACEMENTS[name][1])] += 1
        finally:
            scan.free()
    if name != "host_line":
        assert outcomes["refused"] == 0, outcomes
    elif build[0] == 2:
        assert outcomes["exact"] > 0 and outcomes["refused"] > 0, outcomes   # the [^\w]+ modes keep the scan


# ---- the codes themselves ------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def code_text():
    """tokens at and around the exact/hashed boundary and long ones up to 300 bytes, no two sharing a code"""
    rng = random.Random(31)
    toks = set()
    for n in list(range(1, 17)) + [20, 31, 32, 33, 64, 100, 300]:
        for _ in range(6):
            toks.add(bytes(rng.choice(tc.WORD) for _ in range(n)))
    toks = sorted(toks)
    lines = [b" ".join(toks[i:i + 7]) for i in range(0, len(toks), 7)]
    return b"\n".join(lines) + b"\n", toks


@pytest.mark.parametrize("mode", MODES)
def test_device_codes_equal_the_python_statement(ctx, mode):
    data, toks = code_text()
    want = {key_code(t if mode == tc.TOK_WS else t.lower(), variant(mode)) for t in toks}
    assert sum(c >> 63 for c in want) > 50
    scan = Scan(ctx, data)
    try:
        for kernel, ctas in BUILDS:
            dev.set_option("text_kernel", kernel)
            dev.set_option("text_ctas", ctas)
            try:
                st = scan.count(mode, False, [(0, len(data))])
            finally:
                dev.set_option("text_kernel", 2)
                dev.set_option("text_ctas", 4)
            assert st["flags"] == 0, (kernel, ctas)
            codes, _counts, _reps = scan.tab.fetch()
            assert set(codes.tolist()) == want, (kernel, ctas, len(set(codes.tolist()) ^ want))
    finally:
        scan.free()


def test_field_key_codes_equal_the_python_statement(ctx):
    _data, toks = code_text()
    keys = toks + [b""]
    data = b"".join(k + b",%d\n" % i for i, k in enumerate(keys))
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    tab = ctx.table(16)
    try:
        tab.fields(tb, 0, len(data), (ord(","), 0, dev.FIELD_KEY_STR, 1, dev.OP_SUM_I64))
        st = tab.fields_stats()
        assert st["flags"] == 0 and st["fallback"] == 0
        codes, _acc, _reps = tab.fetch()
        assert set(codes.tolist()) == {key_code(k, "raw", field_key=True) for k in keys}
    finally:
        tb.free()
        tab.free()


# ---- the field fold ------------------------------------------------------------------------------------------------
def field_text(a, b, where, rng):
    """lines key,int,float with a and b as keys `where` apart; returns (text, offset of b's line)"""
    w = tc.Writer(rng)

    def row(k):
        w.line(b"%s,%d,%s,z" % (k, rng.randint(-1000, 1000), repr(rng.uniform(-10, 10)).encode()))
    for i in range(50):
        row(b"k%d" % (i % 7))
    row(a)
    if where == "tiles":
        w.pad_to(2 * tc.F_OWN + 700)
    off = len(w.buf)
    row(b)
    for i in range(50):
        row(b"k%d" % (i % 7) if i % 5 else a)
    return w.data(), off


# (value field, op, record mode): the table folds int sums, minima and maxima and float minima and maxima; float sums
# and mean() (int or float) go through record mode
FIELD_OPS = [(1, dev.OP_SUM_I64, False), (1, dev.OP_MIN_I64, False), (1, dev.OP_MAX_I64, False),
             (2, dev.OP_MIN_F64, False), (2, dev.OP_MAX_F64, False), (1, dev.OP_SUM_I64, True),
             (2, dev.OP_SUM_F64, True)]


@pytest.mark.parametrize("where", ["adjacent", "tiles"])
@pytest.mark.parametrize("kf", [0, -4])
def test_field_fold_flags_colliding_keys(ctx, where, kf):
    rng = random.Random(where + str(kf))
    for i, (a, b, _s, _c) in enumerate(PAIRS["raw"]):
        for control in (False, True):
            data, off = field_text(a, a if control else b, where, rng)
            tb = ctx.textbuf(len(data) + 64)
            tb.upload_all(np.frombuffer(data, dtype=np.uint8))
            tab = ctx.table(14)
            kv = ctx.kv(len(data))
            try:
                for cut, ranges in sorted(cuts(data, off).items()):
                    for vf, op, records in FIELD_OPS:
                        spec = (ord(","), kf, dev.FIELD_KEY_STR, vf, op)
                        tab.clear()
                        for lo, hi in ranges:
                            if records:
                                tab.fields_records(tb, lo, hi, spec, kv)
                            else:
                                tab.fields(tb, lo, hi, spec)
                        flags = tab.fields_stats()["flags"]
                        where_ = (i, control, cut, vf, op, records, flags)
                        if control:
                            assert flags == 0, where_
                        else:
                            assert flags & dev.TF_COLLISION, where_
            finally:
                kv.free()
                tb.free()
                tab.free()


# ---- end to end ----------------------------------------------------------------------------------------------------
@pytest.fixture
def engine(monkeypatch):
    from dampr_b200 import settings, plan
    monkeypatch.setattr(plan, "_BUFFERS", {})
    monkeypatch.setattr(settings, "text_table_log2", settings.text_table_log2)
    yield settings
    plan.release_buffers()


def e2e_text(var, colliding):
    """3000 lines, a on every 97th. b once: on a line after a (colliding), or else on a line with a non-ASCII byte,
    which the [^\\w]+ tokenisers hand to the host"""
    rng = random.Random(var)
    a, b, _s, _c = PAIRS[var][0]
    w = tc.Writer(rng)
    for i in range(3000):
        if i == 700:
            w.line(b"x " + a + b" " + b + b" " + a.upper() if colliding else "\u00e9 ".encode() + b + b" z")
        elif i % 97 == 0:
            w.line(a + b" " + word(rng, 3))
        else:
            w.filler_line()
    return w.data().decode()


def stage_paths():
    from dampr_b200 import runner as runner_mod
    return [how for _s, how, _d in runner_mod.LAST_STATS.stages]


def host_path(caplog):
    hows = stage_paths()
    assert any(how.startswith("host-map") for how in hows), hows
    assert not any("device text" in how for how in hows), hows
    assert any("not lowered (" in r.getMessage() and "collision" in r.getMessage() for r in caplog.records), \
        [r.getMessage() for r in caplog.records]


@pytest.mark.parametrize("idiom,colliding", [("set_rx", True), ("rx", True), ("split", True), ("set_rx", False),
                                             ("rx", False)])
def test_pipelines_over_colliding_tokens_equal_python(engine, tmp_path, caplog, idiom, colliding):
    """colliding: the stage runs on the host and counts like Python; b on a host line only: the device keeps the
    stage, and its counts merged with the host line's equal Python's"""
    from dampr_b200 import Dampr
    text = e2e_text("raw" if idiom == "split" else "sym", colliding)
    P = write_files(tmp_path, [["t.txt", text]])
    fn = {"set_rx": lambda x: set(RX.split(x.lower())), "rx": lambda x: RX.split(x.lower()),
          "split": lambda x: x.split()}[idiom]
    caplog.set_level(logging.WARNING, logger="dampr_b200")
    got = dict(Dampr.text(P).flat_map(fn).count().read())
    exp = collections.Counter()
    with open(P) as f:
        for line in f:
            exp.update(fn(line.rstrip("\n")))
    assert got == dict(exp)
    if colliding:
        host_path(caplog)
    else:
        assert any("device text tokenise+combine" in how for how in stage_paths()), stage_paths()


FIELD_PIPELINES = {
    "sum_i": "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1])).sum()",
    "min_i": "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1])).reduce(min)",
    "max_i": "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: int(l.split(',')[1])).reduce(max)",
    "min_f": "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: float(l.split(',')[2])).reduce(min)",
    "max_f": "Dampr.text(P).a_group_by(lambda l: l.split(',')[-3], lambda l: float(l.split(',')[2])).reduce(max)",
    "sum_f": "Dampr.text(P).a_group_by(lambda l: l.split(',')[0], lambda l: float(l.split(',')[2])).sum()",
    "mean_i": "Dampr.text(P).map(lambda l: l.split(',')).mean(lambda r: r[-3], lambda r: int(r[1]))",
    "mean_f": "Dampr.text(P).map(lambda l: l.split(',')).mean(lambda r: r[0], lambda r: float(r[2]))",
}


def python_field_fold(rows, red):
    groups = collections.defaultdict(list)
    for l in rows:
        f = l.rstrip("\n").split(",")
        groups[f[0]].append(int(f[1]) if red.endswith("_i") else float(f[2]))
    if red.startswith("mean"):
        return {k: sum(v) / float(len(v)) for k, v in groups.items()}
    fold = {"sum": lambda x, y: x + y, "min": min, "max": max}[red[:3]]
    out = {}
    for k, vs in groups.items():
        r = vs[0]
        for v in vs[1:]:
            r = fold(r, v)
        out[k] = r
    return out


@pytest.mark.parametrize("red", sorted(FIELD_PIPELINES))
def test_field_pipelines_over_colliding_keys_equal_python(engine, tmp_path, caplog, red):
    """the same keys without b lower to the field scan; with b the stage runs on the host and equals Python"""
    from dampr_b200 import Dampr
    rng = random.Random(red)
    a, b, _s, _c = PAIRS["raw"][2]
    caplog.set_level(logging.WARNING, logger="dampr_b200")
    for colliding in (False, True):
        rows = []
        for i in range(4000):
            k = a if i % 50 == 0 else (b if i == 3001 and colliding else b"k%d" % rng.randrange(30))
            rows.append("%s,%d,%r\n" % (k.decode(), rng.randint(-10 ** 6, 10 ** 6), rng.uniform(-1e3, 1e3)))
        d = tmp_path / str(colliding)
        d.mkdir()
        P = write_files(d, [["f.csv", "".join(rows)]])
        got = dict(eval(FIELD_PIPELINES[red], {"Dampr": Dampr, "P": P}).read())
        exp = python_field_fold(rows, red)
        if red in ("sum_f", "mean_f"):
            assert got.keys() == exp.keys()       # the host path may add up a key's values in another order
            for k in exp:
                assert got[k] == pytest.approx(exp[k], rel=1e-9, abs=1e-6), k
        else:
            assert got == exp
        if colliding:
            host_path(caplog)
        else:
            assert any("device text fields scan+combine" in how for how in stage_paths()), stage_paths()
