"""The stand-ins of the field-scan kernels (tests/fields_*_standin.py) against CPython, line by line, over the fuzzed
corpora and generated stages of tests/fields_fuzz.py: about 10^5 lines per family (separator byte, split(), JSON)
under stages of every op, plus every one of the 125 separator bytes on small corpora.

A stand-in must be sound: a line it takes is one on which CPython returns the same key code and value bits with every
filter true, a line it drops is one CPython's filters drop before anything raises, every line on which CPython raises
is the host's, and so is every text-mode line holding '\\r'. The stages' kernel arguments are the planner's own
matches (plan._match_text_fields / plan._match_json_fields)."""
import collections
import random

import pytest

import fields_fuzz as fz

# every build of a family (fields_fuzz.builds_of: 18 text, 6 JSON) under cr_is_data off and on, PER_BUILD times, over
# LINES lines each: 72 stages x 1400 lines = about 10^5 lines per family
PER_BUILD, LINES = {"sep": 2, "ws": 2, "json": 6}, 1400
SWEEP_LINES = 400
# at least this share of the generated stages lowered per family, and taken / host lines per build
MIN_LOWERED, MIN_LINES = 0.5, 50


@pytest.fixture(scope="module")
def path(tmp_path_factory):
    p = tmp_path_factory.mktemp("fz") / "f.txt"
    p.write_bytes(b"a,1\n")
    return str(p)


def check_lines(b, data, cr, counts, builds, key=None):
    """every line of data under build b: the stand-in is sound against CPython; tallies the outcomes"""
    for _off, line in fz.lines_of(data):
        got = fz.standin_outcome(b, line, cr)
        py = fz.python_outcome(b.stage, line)
        why = fz.sound(b, line, got, py, cr)
        assert why is None, (b.stage.src, cr, line, got, py, why)
        counts[got[0]] += 1
        if py[0] == fz.HOST:
            counts["py:" + py[1]] += 1
        builds[b.name(), key][got[0]] += 1


def test_found(path):
    """the minimal lines of earlier findings, first"""
    for family, filters, key, value, op, sep, line, cr in fz.FOUND:
        st = fz.Stage(family, None if family == "json" else "lambda l: l.split()" if sep is None else
                      "lambda l: l.split(%r)" % chr(sep), filters, key, value, op)
        assert fz.match(st, path) is not None, st
        b = fz.Build(st)
        got, py = fz.standin_outcome(b, line, cr), fz.python_outcome(st, line)
        assert fz.sound(b, line, got, py, cr) is None, (st.src, line, got, py)


@pytest.mark.parametrize("family", fz.FAMILIES)
def test_standins_are_sound(family, path):
    generated, refused, stages = fz.cover(family, 1, path, PER_BUILD[family])
    counts, builds = collections.Counter(), collections.defaultdict(collections.Counter)
    for j, (b, cr, sep) in enumerate(stages):
        check_lines(b, fz.corpus(family, j, LINES, cr, sep), cr, counts, builds, cr)
    print("\n%s: %d stages generated, %d refused; %s" % (family, generated, refused, dict(sorted(counts.items()))))
    for (name, cr), c in sorted(builds.items()):
        print("  %-22s cr=%d %s" % (name, cr, dict(c)))
    assert generated - refused >= MIN_LOWERED * generated, (generated, refused)
    assert set(builds) == {(name, cr) for name in fz.builds_of(family) for cr in (False, True)}
    assert all(counts[o] > 0 for o in (fz.TAKE, fz.DROP, fz.HOST)), counts
    per_build = collections.defaultdict(collections.Counter)
    for (name, _cr), c in builds.items():
        per_build[name].update(c)
    for name, c in per_build.items():   # every build reaches both sides of its decision
        assert c[fz.TAKE] >= MIN_LINES and c[fz.HOST] >= MIN_LINES, (name, c)
        assert "where" not in name or c[fz.DROP] >= MIN_LINES, (name, c)


def test_every_separator_byte(path):
    """all 125 separator bytes, two stages each (one plain, one with filters where the generator gives one)"""
    counts, builds = collections.Counter(), collections.defaultdict(collections.Counter)
    for sep in fz.SEPS:
        data = fz.corpus("sep", 5000 + sep, SWEEP_LINES, sep % 2 == 0, sep)
        sts, _n = fz.gen_stages(9000 + sep, "sep", 6, path, sep)
        kinds = {}
        for st in sts:
            kinds.setdefault(bool(st.filters), st)
        for st in kinds.values():
            check_lines(fz.Build(st), data, sep % 2 == 0, counts, builds)
    print("\nseparator sweep: %s" % dict(sorted(counts.items())))
    assert counts[fz.TAKE] > 10000 and counts[fz.DROP] > 1000 and counts[fz.HOST] > 10000, counts


def test_the_corpus_is_the_seeds():
    for family in fz.FAMILIES:
        a = fz.corpus(family, 3, 3000, True, ord(";"))
        assert a == fz.corpus(family, 3, 3000, True, ord(";"))
        assert a != fz.corpus(family, 4, 3000, True, ord(";"))

    def stages(seed):
        rng = random.Random(seed)
        return [fz.gen_stage(rng, f, ord(",")).src for f in fz.FAMILIES for _ in range(20)]
    assert stages(5) == stages(5) != stages(6)
