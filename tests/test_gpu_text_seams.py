"""The text kernels (csrc/text2.cu in its 4-, 3- and 2-CTA builds, csrc/text.cu, csrc/fields.cu) on corpora that sit
on their structural seams (tests/text_contract.py), under the whole ownership range, random 16-byte-aligned cuts and
cuts at strip and tile multiples +- 16. Every call is either exactly right or says it is not: the flags lie between
what the contract requires and what it allows, and without a refusal flag the fallback list, the table and the
line, '' and folded counters equal plain Python over the lines the device kept."""
import functools

import numpy as np
import pytest

import text_contract as tc
from dampr_b200 import device as dev
from dampr_b200 import keycodes

pytestmark = pytest.mark.gpu

BUILDS = [(2, 4), (2, 3), (2, 2), (1, 2)]
REFUSE = tc.TF_NONASCII | tc.TF_LONGLINE | tc.TF_TABLEFULL


@pytest.fixture(params=BUILDS, ids=["v2-4cta", "v2-3cta", "v2-2cta", "v1"])
def build(request):
    dev.set_option("text_kernel", request.param[0])
    dev.set_option("text_ctas", request.param[1])
    try:
        yield request.param
    finally:
        dev.set_option("text_kernel", 2)
        dev.set_option("text_ctas", 4)


@functools.lru_cache(maxsize=None)
def corpus(name):
    if name.startswith("A"):
        return tc.set_history_corpus(int(name[1:]))[0]
    return {"B": lambda: tc.token_seam_corpus()[0], "C": lambda: tc.long_token_corpus()[0],
            "D8": lambda: tc.bad_line_corpus(max_bad=8)[0], "D9": lambda: tc.bad_line_corpus(max_bad=9)[0]}[name]()


@functools.lru_cache(maxsize=None)
def expectation(name, kernel, mode, cr_is_data):
    data = corpus(name)
    fb = tc.expected_fallback(data, kernel, mode, cr_is_data)
    return fb, tc.expected_table(data, mode, cr_is_data, fb)


class Scan(object):
    """one uploaded text and one table, cleared before every scan"""

    def __init__(self, ctx, data):
        self.data = data
        self.tb = ctx.textbuf(len(data) + 64)
        self.tb.upload_all(np.frombuffer(data, dtype=np.uint8) if data else np.zeros(0, np.uint8))
        self.tab = ctx.table(18)

    def count(self, mode, cr_is_data, ranges):
        self.tab.clear()
        for lo, hi in ranges:
            self.tab.count(self.tb, lo, hi, mode, cr_is_data)
        return self.tab.stats()

    def table(self, mode):
        codes, counts, reps = self.tab.fetch()
        words = keycodes.decode_table(codes, reps, mode, lambda o, n: self.data[o:o + n])
        got = dict(zip(words, counts.tolist()))
        assert len(got) == len(words), "two table entries decoded to the same word"
        return got

    def free(self):
        self.tb.free()
        self.tab.free()


def check_count(scan, name, build, mode, cr_is_data, cut, ranges, must_be_clean=False):
    """one scan against the contract; returns True when the device refused (the scan is the caller's)"""
    kernel, ctas = build
    data = scan.data
    st = scan.count(mode, cr_is_data, ranges)
    req, allowed = tc.refusals(data, mode, cr_is_data, ranges, kernel, ctas)
    where = (name, build, mode, cr_is_data, cut)
    flags = st["flags"]
    assert flags & req == req and flags & ~allowed == 0, (where, flags, req, allowed)
    if must_be_clean:
        assert flags == 0, where
    if flags & REFUSE:
        return True
    fb, exp = expectation(name, kernel, mode, cr_is_data)
    assert sorted(scan.tab.fallback_lines().tolist()) == fb, where
    assert st["fallback"] == len(fb), where
    got = scan.table(mode)
    assert got == exp["table"], (where, sorted(set(got.items()) ^ set(exp["table"].items()))[:10])
    assert st["lines"] == exp["lines"] and st["folded"] == exp["folded"], (where, st, exp["lines"], exp["folded"])
    if mode != tc.TOK_WS:
        assert st["empty"] == exp["empty"], (where, st["empty"], exp["empty"])
    return False


def run_corpus(ctx, name, build, modes, crs=(False, True), clean=lambda mode, cr: False):
    data = corpus(name)
    scan = Scan(ctx, data)
    try:
        for cut, ranges in sorted(tc.cut_sets(len(data)).items()):
            for mode in modes:
                for cr in crs:
                    check_count(scan, name, build, mode, cr, cut, ranges, clean(mode, cr) and cut == "whole")
    finally:
        scan.free()


# ---- A: the set() history of a line that straddles a round ----------------------------------------------------------
@pytest.mark.parametrize("D", tc.D_VALUES)
def test_set_history_lines(ctx, build, D):
    """D distinct tokens, each written twice in other cases: v2 with D <= HCAP exact and flag-free, above HCAP exact
    or TF_LONGLINE; v1 exact; the non-set mode exact and flag-free everywhere"""
    kernel, ctas = build
    run_corpus(ctx, "A%d" % D, build, (tc.TOK_NONWORD_LOWER_SET,), crs=(False,),
               clean=lambda m, cr: kernel == 1 or D <= tc.HCAP[ctas])
    run_corpus(ctx, "A%d" % D, build, (tc.TOK_NONWORD_LOWER, tc.TOK_WS), crs=(False,), clean=lambda m, cr: True)


# ---- B: exact/hashed key boundary at every alignment and seam ---------------------------------------------------------
def test_token_seams(ctx, build):
    run_corpus(ctx, "B", build, (tc.TOK_WS, tc.TOK_NONWORD_LOWER_SET, tc.TOK_NONWORD_LOWER),
               clean=lambda m, cr: build[0] == 2 or m == tc.TOK_WS)


def test_nul_token_does_not_merge_with_its_prefix(ctx, build):
    """str.split: a NUL inside a short token forces the hashed code; "a\\0" and "a" are two words"""
    data = b"a\0 a a\0 \0a a\x7f ab\0cd abcd\n" * 3
    scan = Scan(ctx, data)
    try:
        st = scan.count(tc.TOK_WS, False, [(0, len(data))])
        assert st["flags"] == 0
        assert scan.table(tc.TOK_WS) == {"a\0": 6, "a": 3, "\0a": 3, "a\x7f": 3, "ab\0cd": 3, "abcd": 3}
    finally:
        scan.free()


# ---- C: the str.split long-token combiner ---------------------------------------------------------------------------
def test_long_tokens_through_the_combiner(ctx, build):
    """~5,000 tokens of 10-40 bytes with shared prefixes, last-byte twins and one-byte extensions: exact counts and
    no false TF_COLLISION; the v1 build's verify pass leaves the flags at 0 too"""
    data = corpus("C")
    scan = Scan(ctx, data)
    try:
        for cut, ranges in sorted(tc.cut_sets(len(data)).items()):
            check_count(scan, "C", build, tc.TOK_WS, False, cut, ranges, must_be_clean=True)
            if build[0] == 1:
                scan.tab.verify(scan.tb, 0, len(data), tc.TOK_WS)
                assert scan.tab.stats()["flags"] == 0, cut
    finally:
        scan.free()


# ---- D: the per-line fallback ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["D8", "D9"])
def test_per_line_fallback(ctx, build, name):
    """0-8 (D8) or 0-9 (D9) host lines per strip: with at most 8 per strip the list is exact and the flags 0"""
    run_corpus(ctx, name, build, (tc.TOK_NONWORD_LOWER_SET, tc.TOK_NONWORD_LOWER, tc.TOK_WS),
               clean=lambda m, cr: build[0] == 2 and name == "D8" and m != tc.TOK_WS)


# ---- E: the field fold -----------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def fields_data(sep, longest):
    return tc.fields_corpus(sep, longest=longest)[0]


def check_fields(ctx, tb, tab, data, spec, cr_is_data, cut, ranges):
    sep, kf, kind, vf, op = spec
    tab.clear()
    for lo, hi in ranges:
        tab.fields(tb, lo, hi, spec, cr_is_data)
    st = tab.fields_stats()
    exp = tc.fields_prediction(data, spec, cr_is_data)
    where = (spec, cr_is_data, cut)
    assert st["flags"] == exp["flags"], (where, st)
    if exp["flags"]:
        return
    assert sorted(tab.fallback_lines().tolist()) == exp["fallback"], where
    assert (st["lines"], st["folded"], st["max_abs"]) == (exp["lines"], exp["folded"], exp["max_abs"]), (where, st)
    if kind == tc.FIELD_KEY_INT:
        codes, vals = tab.fields_fetch(op)
        got = dict(zip((codes ^ np.uint64(1 << 63)).view(np.int64).tolist(), vals.tolist()))
    else:
        words, acc, codes, reps = tab.fetch_words(tb, dev.TOK_WS, 64)
        keys = []
        for w, c, r in zip(words.tolist(), codes.tolist(), reps.tolist()):
            k = data[(r >> 20):(r >> 20) + (r & 0xFFFFF)] if c >> 63 else w
            assert w == k[:64], (where, k)   # hashed keys are read back from their representative, truncated
            keys.append(k.decode("ascii"))
        got = dict(zip(keys, dev.decode_fold(acc, op).tolist()))
        assert len(got) == len(words)
    assert got == exp["table"], (where, sorted(set(got.items()) ^ set(exp["table"].items()))[:10])


@pytest.mark.parametrize("sep", tc.FIELD_SEPS)
def test_field_fold(ctx, sep):
    data = fields_data(sep, tc.F_FB_MAXLEN)
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    tab = ctx.table(18)
    try:
        for cut, ranges in sorted(tc.cut_sets(len(data)).items()):
            for i, (kf, kind, vf, op) in enumerate(tc.FIELD_SPECS):
                for cr in (False, True):
                    if cut != "whole" and (i + cr) % 3:
                        continue   # every spec and both '\r' rules over the whole range, a third of them per split
                    check_fields(ctx, tb, tab, data, (sep, kf, kind, vf, op), cr, cut, ranges)
    finally:
        tb.free()
        tab.free()


def test_field_line_of_64k_ends_the_scan(ctx):
    data = fields_data(ord(","), tc.F_FB_MAXLEN + 1)
    tb = ctx.textbuf(len(data) + 64)
    tb.upload_all(np.frombuffer(data, dtype=np.uint8))
    tab = ctx.table(18)
    try:
        for cut, ranges in sorted(tc.cut_sets(len(data)).items()):
            check_fields(ctx, tb, tab, data, (ord(","), 0, tc.FIELD_KEY_STR, tc.FIELD_VAL_ONE, tc.OP_SUM_I64), False,
                         cut, ranges)
    finally:
        tb.free()
        tab.free()


# ---- F: key decoding on the device -----------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [tc.TOK_WS, tc.TOK_NONWORD_LOWER_SET, tc.TOK_NONWORD_LOWER])
def test_fetch_words_and_kv_decode_at_every_width(ctx, mode):
    data = corpus("B")
    scan = Scan(ctx, data)
    try:
        st = scan.count(mode, False, [(0, len(data))])
        assert st["flags"] == 0 and st["hashed"] > 0
        codes, counts, reps = scan.tab.fetch()
        full = dict(zip(codes.tolist(), (w.encode("ascii") for w in
                                         keycodes.decode_table(codes, reps, mode, lambda o, n: data[o:o + n]))))
        assert any(c >> 63 and len(full[c]) > 16 for c in full)     # hashed tokens longer than the narrowest width
        kv = scan.tab.to_kv()
        keys, _vals = kv.columns()
        for width in (16, 24, 32, 64, 256):
            words, wcounts, wcodes, wreps = scan.tab.fetch_words(scan.tb, mode, width)
            assert sorted(wcodes.tolist()) == sorted(full)
            for w, c in zip(words.tolist(), wcodes.tolist()):
                assert w == full[c][:width].rstrip(b"\0"), (width, c)
            kw = kv.decode_words(mode, width)
            for w, c in zip(kw.tolist(), keys.tolist()):
                assert w == (b"" if c >> 63 else full[c][:width].rstrip(b"\0")), (width, c)
        kv.free()
    finally:
        scan.free()


# ---- G: end to end down the planner's retry ladder ------------------------------------------------------------------
def test_docfreq_down_the_retry_ladder(ctx, tmp_path):
    """lines with up to 257 distinct tokens: the 4- and 2-CTA builds refuse (TF_LONGLINE), the planner retries down
    to the first-generation kernel and still reports a device scan equal to the reference"""
    import re
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    from oracle import refsem
    data = b"".join(corpus("A%d" % d) for d in (31, 65, 129, 257))
    scan = Scan(ctx, data)
    try:
        for ctas in (4, 2):
            dev.set_option("text_ctas", ctas)
            try:
                assert scan.count(tc.TOK_NONWORD_LOWER_SET, False, [(0, len(data))])["flags"] & tc.TF_LONGLINE
            finally:
                dev.set_option("text_ctas", 4)
    finally:
        scan.free()
    p = tmp_path / "a.txt"
    p.write_bytes(data)
    RX = re.compile(r"[^\w]+")
    got = Dampr.text(str(p)).flat_map(lambda x: set(RX.split(x.lower()))).count().read()
    assert any("device text tokenise+combine" in how for _s, how, _d in runner_mod.LAST_STATS.stages)
    assert dict(got) == dict(refsem.docfreq(data)[0])
