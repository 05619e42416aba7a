"""CPU checks of tests/text_contract.py: the corpora reach the seams the GPU suite is meant to pin, and the contract
oracle composes back to the reference semantics (expected device table + Python over the expected host lines ==
Python over the whole text). Needs no native library."""
import bisect
import functools
import gzip

import pytest

import text_contract as tc
from oracle import refsem
from fields_standin import python_fold

MODES = (tc.TOK_WS, tc.TOK_NONWORD_LOWER_SET, tc.TOK_NONWORD_LOWER)


@functools.lru_cache(maxsize=None)
def corpus(name):
    if name.startswith("A"):
        return tc.set_history_corpus(int(name[1:]))[0]
    return {"B": lambda: tc.token_seam_corpus()[0], "C": lambda: tc.long_token_corpus()[0],
            "D8": lambda: tc.bad_line_corpus(max_bad=8)[0], "D9": lambda: tc.bad_line_corpus(max_bad=9)[0]}[name]()


TEXT_CORPORA = ["A%d" % d for d in (31, 64, 129, 257)] + ["B", "C", "D8", "D9"]


def reference(data, mode, cr_is_data):
    """{token: count} (with '') and the line count of the reference run over the whole text"""
    if not cr_is_data:
        if mode == tc.TOK_WS:
            c = refsem.wc_counts(data)
        elif mode == tc.TOK_NONWORD_LOWER_SET:
            c = refsem.docfreq(data)[0]
        else:
            c = refsem.termfreq_nonset(data)
        return dict(c), len(refsem.text_lines(data))
    t, e, n = tc.python_over_lines(data, [o for o, _ in tc.nl_lines(data)], mode, True)
    if e:
        t[""] = e
    return t, n


@pytest.mark.parametrize("name", TEXT_CORPORA)
@pytest.mark.parametrize("cr_is_data", [False, True])
def test_text_oracle_composes_to_the_reference(name, cr_is_data):
    data = corpus(name)
    for mode in MODES:
        fb = tc.expected_fallback(data, 2, mode, cr_is_data)
        if any(c >= 0x80 for c in data) and mode == tc.TOK_WS:
            continue   # str.split mode refuses non-ASCII text as a whole
        exp = tc.expected_table(data, mode, cr_is_data, fb)
        host, host_empty, host_lines = tc.python_over_lines(data, [e >> 16 for e in fb], mode, cr_is_data)
        got = dict(exp["table"])
        for k, v in host.items():
            got[k] = got.get(k, 0) + v
        ref, ref_lines = reference(data, mode, cr_is_data)
        ref_empty = ref.pop("", 0)
        assert got == ref, (name, mode)
        if mode != tc.TOK_WS:
            assert exp["empty"] + host_empty == ref_empty
            assert exp["lines"] + host_lines == ref_lines
        # every listed line is a whole '\n' line of the text
        for e in fb:
            o, ln = e >> 16, e & 0xFFFF
            assert (o == 0 or data[o - 1:o] == b"\n") and data[o + ln:o + ln + 1] in (b"\n", b"")


def _straddled(data, seams):
    starts = set(o for o, _ in tc.nl_lines(data))
    return [s for s in seams if s not in starts and s < len(data)]


@pytest.mark.parametrize("name", ["A31", "A257", "B", "D8"])
def test_lines_straddle_every_strip_and_tile_seam(name):
    data = corpus(name)
    seams = list(range(tc.V_STRIP, len(data), tc.V_STRIP))
    assert len(seams) >= 8 and any(s % tc.V_OWN == 0 for s in seams)
    assert _straddled(data, seams) == seams


def test_token_lengths_and_alignments_cross_the_seams():
    data, planted = tc.token_seam_corpus()
    toks = [(m.start(), m.end() - m.start()) for m in tc.WS_TOKEN.finditer(data)]
    n = len(data)

    def crossing(seams):
        seams = sorted(seams)
        out = set()
        for st, ln in toks:
            i = bisect.bisect_right(seams, st)
            if i < len(seams) and seams[i] < st + ln:
                out.add((ln, st % 4))
        return out
    need = set((L, a) for L in range(8, 14) for a in range(4))
    tile = [s for s in range(tc.V_OWN, n, tc.V_OWN)]
    strip = [s for s in range(tc.V_STRIP, n, tc.V_STRIP) if s % tc.V_OWN]
    win_end = [t + tc.V_WIN_END for t in range(0, n - tc.V_WIN_END, tc.V_OWN)]
    assert need <= crossing(tile)
    assert need <= crossing(strip)
    assert need <= crossing(win_end)
    # ... and tokens of 1-16, 40 and 200 bytes end on a seam, some of 5000 bytes exist, NUL / DEL sit inside tokens
    lens = set(ln for st, ln in toks if (st + ln) % tc.V_STRIP == 0)
    assert set(range(1, 17)) | {40, 200} <= lens
    assert any(ln == 5000 for _s, ln in toks)
    words = set(data[s:s + ln] for s, ln in toks)
    assert {b"a", b"a\0", b"\0a", b"a\x7f"} <= words
    assert any(b"\0" in w and 8 <= len(w) <= 13 for w in words)
    # every str.split whitespace byte but '\n' / '\r' separates tokens here ('\r' is in the per-line corpus)
    for b in b"\t\x0b\x0c\x1c\x1d\x1e\x1f ":
        assert bytes([b]) in data


@pytest.mark.parametrize("D", tc.D_VALUES)
def test_set_lines_hold_d_distinct_tokens_twice(D):
    data, big = tc.set_history_corpus(D)
    assert len(big) >= 8
    for o, ln in big:
        line = data[o:o + ln]
        toks = [t for t in tc.RX.split(line.decode("ascii").lower()) if t]
        assert len(set(toks)) == D and len(toks) >= 2 * D
        assert 300 <= ln <= 1900, ln
        assert any(t != t.lower() for t in tc.RX.split(line.decode("ascii")))   # case variants
    near = [o for o, _ in big if (-o) % tc.V_STRIP <= 100]
    assert near and any((-o) % tc.V_OWN <= 100 for o in near)


def test_strips_with_eight_and_nine_host_lines():
    for max_bad, must in ((8, 8), (9, 9)):
        data = corpus("D%d" % max_bad)
        per = {}
        for o, ln in tc.nl_lines(data):
            if tc.line_is_bad(data[o:o + ln], False):
                per[o // tc.V_STRIP] = per.get(o // tc.V_STRIP, 0) + 1
        assert max(per.values()) == must
        assert set(range(0, must + 1)) - {0} <= set(per.values())
    data = corpus("D8")
    assert tc.line_is_bad(data[data.rfind(b"\n") + 1:], True) and not data.endswith(b"\n")
    assert b"\r\n" in data and any(data[i + 1] not in b"\n" for i in range(len(data) - 1) if data[i] == 13)
    # bad lines that straddle a strip seam
    bad_cross = [o for o, ln in tc.nl_lines(data) if tc.line_is_bad(data[o:o + ln], False)
                 and o // tc.V_STRIP != (o + ln) // tc.V_STRIP]
    assert len(bad_cross) >= 3


@functools.lru_cache(maxsize=None)
def fields_corpus(sep, longest=tc.F_FB_MAXLEN):
    return tc.fields_corpus(sep, longest=longest)


def test_field_line_lengths_at_tile_seams():
    for longest in (tc.F_FB_MAXLEN, tc.F_FB_MAXLEN + 1):
        data, longs = fields_corpus(ord(","), longest)
        lens = dict((o, ln) for o, ln in tc.nl_lines(data))
        for L in (4094, 4095, 4096, 4097, longest):
            o = longs[L]
            assert lens[o] == L
            assert o // tc.F_OWN != (o + L) // tc.F_OWN     # it straddles a tile seam
    data, _ = fields_corpus(ord(","))
    assert not data.endswith(b"\n")


@pytest.mark.parametrize("sep", tc.FIELD_SEPS)
@pytest.mark.parametrize("cr_is_data", [False, True])
def test_fields_oracle_composes_to_python_fold(sep, cr_is_data, tmp_path):
    data, _ = fields_corpus(sep)
    p = str(tmp_path / ("f.csv.gz" if cr_is_data else "f.csv"))
    if cr_is_data:
        with gzip.open(p, "wb") as f:
            f.write(data)
    else:
        with open(p, "wb") as f:
            f.write(data)
    for kf, kind, vf, op in tc.FIELD_SPECS:
        spec = (sep, kf, kind, vf, op)
        exp = tc.fields_prediction(data, spec, cr_is_data)
        assert exp["flags"] == 0 and exp["lines"] > 0
        host = {}
        for e in exp["fallback"]:
            o, ln = e >> 16, e & 0xFFFF
            for k, v in tc.python_fold_lines(tc.host_lines(data[o:o + ln], cr_is_data), spec).items():
                host[k] = tc.fold(op, host[k], v) if k in host else v
        got = dict(exp["table"])
        for k, v in host.items():
            got[k] = tc.fold(op, got[k], v) if k in got else v
        if op == tc.OP_SUM_I64:
            got = dict((k, tc.wrap64(v)) for k, v in got.items())
        key, value = tc.field_functions(spec)
        want = python_fold(p, key, value, lambda a, b: tc.fold(op, a, b))
        if op == tc.OP_SUM_I64:
            want = sorted(repr((k, tc.wrap64(v))) for k, v in (eval(r) for r in want))
        assert sorted(repr(x) for x in got.items()) == want, spec
        # the spellings int() takes but the device does not are exactly the host's
        assert all(tc.field_line_to_host(data[(e >> 16):(e >> 16) + (e & 0xFFFF)], spec, cr_is_data)
                   for e in exp["fallback"])


def test_field_refusals():
    data, _ = fields_corpus(ord(","), tc.F_FB_MAXLEN + 1)
    exp = tc.fields_prediction(data, (ord(","), 0, tc.FIELD_KEY_STR, tc.FIELD_VAL_ONE, tc.OP_SUM_I64), False)
    assert exp["flags"] == tc.TF_LONGLINE
    data, longs = fields_corpus(ord(","))
    exp = tc.fields_prediction(data, (ord(","), 0, tc.FIELD_KEY_STR, tc.FIELD_VAL_ONE, tc.OP_SUM_I64), False)
    fb = dict((e >> 16, e & 0xFFFF) for e in exp["fallback"])
    assert fb[longs[tc.F_FB_MAXLEN]] == tc.F_FB_MAXLEN and fb[longs[4096]] == 4096 and longs[4095] not in fb
    # int() spellings: 18 digits are the device's, 19 digits and the rest are Python's
    for s, dev in [(b"0", True), (b"-0", True), (b"+0", True), (b"007", True), (b"9" * 18, True), (b"-" + b"9" * 18, True),
                   (b"1" + b"0" * 18, False), (b"+", False), (b"-", False), (b"", False), (b"5_0", False), (b" 5", False),
                   (b"5 ", False), (b"0x10", False)]:
        assert tc.field_line_to_host(b"k," + s, (ord(","), 0, tc.FIELD_KEY_STR, 1, tc.OP_SUM_I64), False) != dev, s


def test_refusal_prediction_follows_the_ownership_split():
    data, _ = tc.bad_line_corpus(max_bad=8)
    n = len(data)
    assert tc.refusals(data, tc.TOK_NONWORD_LOWER_SET, False, [(0, n)], 2) == (0, 0)
    assert tc.refusals(data, tc.TOK_NONWORD_LOWER_SET, True, [(0, n)], 2) == (0, 0)
    data9, _ = tc.bad_line_corpus(max_bad=9)
    assert tc.refusals(data9, tc.TOK_NONWORD_LOWER, False, [(0, len(data9))], 2)[0] == tc.TF_NONASCII
    assert tc.refusals(data, tc.TOK_NONWORD_LOWER, False, [(0, n)], 1)[0] == tc.TF_NONASCII | tc.TF_CR
    a = tc.set_history_corpus(65)[0]
    assert tc.refusals(a, tc.TOK_NONWORD_LOWER_SET, False, [(0, len(a))], 2, 4) == (0, tc.TF_LONGLINE)
    assert tc.refusals(a, tc.TOK_NONWORD_LOWER_SET, False, [(0, len(a))], 2, 3) == (0, 0)
    assert tc.refusals(a, tc.TOK_NONWORD_LOWER, False, [(0, len(a))], 2, 4) == (0, 0)
    for cuts in tc.cut_sets(n).values():
        assert cuts[0][0] == 0 and cuts[-1][1] == n and all(lo % 16 == 0 for lo, _ in cuts)
        assert all(a[1] == b[0] for a, b in zip(cuts, cuts[1:]))
