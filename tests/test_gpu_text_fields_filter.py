"""Filter programs on the device (the WHERE builds of csrc/fields.cu with and / or / not, string tests and whole-line
tests): the reference pipelines of tests/test_text_fields_filter_lowering.py, every field-scan family (separator byte,
split(), JSON, tuple keys, computed values) in table and record modes against plain Python, .gz CRLF rows and text-mode
CR lines, needles across the 16 KB tile seam and in 4 KB lines, non-ASCII lines and needles, undecided leaves on both
sides of `and` / `or`, a NaN under `not`, and random programs of 1 .. 8 leaves against Python. Each case asserts
the stage's path."""
import json
import math
import random

import pytest

from fields_standin import python_lines, reference_outputs, write_files
from test_text_fields_filter_lowering import GOLDEN, HEADER, NEEDLE, PIPELINES, datasets

pytestmark = pytest.mark.gpu


@pytest.fixture
def engine(monkeypatch):
    from dampr_b200 import settings, plan
    monkeypatch.setattr(plan, "_BUFFERS", {})
    yield settings
    plan.release_buffers()


def run(src, P):
    from dampr_b200 import Dampr
    from dampr_b200 import runner as runner_mod
    got = sorted(repr(x) for x in eval(src, {"Dampr": Dampr, "P": P, "json": json}).run())
    return got, runner_mod.LAST_STATS.stages[0]


def python_run(src, P):
    """the pipeline in plain Python: Dampr's text / json / map / filter / keyed folds over python_lines"""
    class Q(object):
        def __init__(self, rows):
            self.rows = rows

        def map(self, f):
            return Q([f(x) for x in self.rows])

        def filter(self, f):
            return Q([x for x in self.rows if f(x)])

        def _fold(self, k, v, b):
            out = {}
            for x in self.rows:
                kk, vv = k(x), v(x)
                out[kk] = b(out[kk], vv) if kk in out else vv
            return out

        def count(self, k):
            return sorted(repr(x) for x in self._fold(k, lambda x: 1, lambda a, b: a + b).items())

        def a_group_by(self, k, v):
            q = self

            class G(object):
                def sum(self):
                    return sorted(repr(x) for x in q._fold(k, v, lambda a, b: a + b).items())

                def reduce(self, f):
                    return sorted(repr(x) for x in q._fold(k, v, f).items())
            return G()

        def mean(self, k, v):
            out = self._fold(k, lambda x: (v(x), 1), lambda a, b: (a[0] + b[0], a[1] + b[1]))
            return sorted(repr((kk, s / c)) for kk, (s, c) in out.items())

    class D(object):
        @staticmethod
        def text(p):
            return Q(python_lines(p))

        @staticmethod
        def json(p):
            return Q([json.loads(l) for l in python_lines(p)])
    return eval(src.replace(".run()", ""), {"Dampr": D, "P": P, "json": json})


def same(got, exp):
    """equal records; float sums and means within 2^-40 relative"""
    val = {"nan": float("nan"), "inf": float("inf")}
    g, e = [eval(x, dict(val)) for x in got], [eval(x, dict(val)) for x in exp]
    assert [k for k, _ in g] == [k for k, _ in e], (got[:5], exp[:5])
    for (k, gv), (_k, ev) in zip(g, e):
        if type(ev) is float and not math.isnan(ev):
            assert abs(gv - ev) <= 2.0 ** -40 * max(1.0, abs(ev)), (k, gv, ev)
        else:
            assert repr(gv) == repr(ev), (k, gv, ev)


def check(src, P, host_lines=None, filtered=None, detail=()):
    got, (_s, how, d) = run(src, P)
    same(got, python_run(src, P))
    assert NEEDLE in how, (src, how, d)
    if host_lines is not None:
        assert "host_lines=%d" % host_lines in d, (src, d)
    if filtered is not None:
        assert "filtered=%d" % filtered in d, (src, d)
    for x in detail:
        assert x in d, (src, d)
    return d


@pytest.mark.parametrize("name", sorted(PIPELINES))
def test_reference_pipelines(name, engine, tmp_path):
    files = datasets()[name]
    P = write_files(tmp_path, files)
    for src, exp in zip(PIPELINES[name], reference_outputs(files, PIPELINES[name], GOLDEN)):
        got, (_s, how, d) = run(src, P)
        same(got, exp)
        assert NEEDLE in how and "filtered=" in d, (src, how, d)


def clean_log(n, seed, sep=","):
    rng = random.Random(seed)
    rows = [sep.join(HEADER.split(","))] if sep != " " else []
    for i in range(n):
        rows.append(sep.join([str(rng.randrange(50)), rng.choice(["GET", "POST", "PUT"]),
                              str(rng.choice([200, 301, 404, 500, 503])), str(rng.randrange(0, 9000)),
                              rng.choice(["0.25", "1e-3", "2.5", "nan"]), rng.choice(["a", "bb", "ERRORx", "timeout"]),
                              rng.choice(["/api/users", "/api/x", "/static/a.js", "/x", "/"])]))
        if rng.random() < 0.05:
            rows.append("# comment %d" % i)
    return "".join(r + "\n" for r in rows)


def test_the_issue_examples(engine, tmp_path):
    P = write_files(tmp_path, [["log.txt", clean_log(20000, 1, " ").replace("# comment", "#comment")]])
    check("Dampr.text(P).filter(lambda l: 'ERROR' in l).map(lambda l: l.split()).count(lambda r: r[3])", P,
          host_lines=0, detail=["sep=ws"])
    P = write_files(tmp_path, [["log.csv", clean_log(20000, 2)]])
    check("Dampr.text(P).filter(lambda l: not l.startswith('#')).map(lambda l: l.split(','))"
          ".filter(lambda r: r[1] == 'GET' and (int(r[2]) >= 500 or r[6].startswith('/api/')))"
          ".a_group_by(lambda r: r[0], lambda r: int(r[3])).sum()", P, host_lines=0)
    check("Dampr.text(P).filter(lambda l: not l.startswith('#') and l != '" + HEADER + "').map(lambda l: l.split(','))"
          ".filter(lambda r: r[1] == 'GET' and (int(r[2]) >= 500 or r[6].startswith('/api/')))"
          ".a_group_by(lambda r: r[0], lambda r: int(r[3])).sum()", P, host_lines=0)
    rng = random.Random(3)
    recs = [{"level": rng.choice(["ERROR", "WARN", "INFO"]), "msg": rng.choice(["a timeout b", "ok", "timeout"]),
             "svc": rng.choice(["s1", "s2", "s3"])} for _ in range(20000)]
    P = write_files(tmp_path, [["j.jsonl", "".join(json.dumps(r) + "\n" for r in recs)]])
    check("Dampr.json(P).filter(lambda r: r['level'] in ('ERROR', 'WARN') or 'timeout' in r['msg'])"
          ".count(lambda r: r['svc'])", P, host_lines=0, detail=["sep=json"])


FAMILIES = [
    # separator byte, int / float values, table and record modes
    "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: len(r) == 7 and (r[5].endswith('x') or "
    "'api' in r[6]) and not r[1] == 'PUT').a_group_by(lambda r: r[1], lambda r: int(r[3])).reduce(max)",
    "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: len(r) == 7 and r[0] != 'ts' and "
    "(len(r[5]) > 2 or r[6].startswith(('/x', '/static')))).mean(lambda r: r[1], lambda r: int(r[3]))",
    "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: len(r) == 7 and r[0] != 'ts' and "
    "not (float(r[4]) < 1.0) or r[0] == 'x').a_group_by(lambda r: r[5], lambda r: float(r[4])).sum()",
    # tuple key and computed value
    "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: len(r) == 7 and r[0] != 'ts' and "
    "r[6].strip() and not r[6].endswith('/')).count(lambda r: (r[1], int(r[2])))",
    "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: len(r) == 7 and r[0] != 'ts' and "
    "('ERROR' in r[5] or int(r[2]) >= 500)).a_group_by(lambda r: r[1], lambda r: int(r[3]) * 2).sum()",
    # whole line in front of the split
    "Dampr.text(P).filter(lambda l: not l.startswith('#') and len(l) > 20 and l.strip() and l != '" + HEADER + "')"
    ".map(lambda l: l.split(',')).filter(lambda r: r[6] in ('/', '/x') or not 'a' in r[5])"
    ".a_group_by(lambda r: r[0], lambda r: float(r[4])).sum()",
]


@pytest.mark.parametrize("gz", [False, True])
def test_every_family(gz, engine, tmp_path):
    text = clean_log(30000, 4)
    P = write_files(tmp_path, [["l.csv.gz" if gz else "l.csv", text]])
    for src in FAMILIES:
        check(src, P)
    T = write_files(tmp_path, [["t.tsv", text.replace(",", "\t")]])
    check("Dampr.text(P).map(lambda l: l.split('\\t')).filter(lambda r: len(r) == 7 and (r[1] == 'GET' or "
          "r[6].endswith('.js'))).count(lambda r: r[5])", T, host_lines=0)
    W = write_files(tmp_path, [["w.txt", text.replace(",", "  ")]])
    check("Dampr.text(P).map(lambda l: l.split()).filter(lambda r: len(r) == 7 and not (r[1] == 'GET' or "
          "r[6].startswith('/api')) and len(r[5]) < 5).count(lambda r: r[1])", W, host_lines=0, detail=["sep=ws"])


def test_crlf_and_cr(engine, tmp_path):
    """.gz keeps '\\r' as data: endswith('x') is False and strip() removes it; text mode hands CR lines to the host"""
    rows = ["a,x", "b,x\r", "c,y\r", "\r", "d,x", " \r"]
    text = "".join(r + "\n" for r in rows * 500)
    src = "Dampr.text(P).filter(lambda l: l.strip() and (l.endswith('x') or l.startswith('c')))" \
          ".count(lambda l: l.split(',')[0])"
    G = write_files(tmp_path, [["c.csv.gz", text]])
    check(src, G, host_lines=0)
    T = write_files(tmp_path, [["c.csv", text]])
    d = check(src, T)
    assert "host_lines=0" not in d


def test_seams_long_lines_and_needles(engine, tmp_path):
    rng = random.Random(5)
    rows = []
    for i in range(3000):
        k = rng.choice([1, 40, 500, 4000, 4094, 4095, 4200])
        body = "".join(rng.choice("abcxyz") for _ in range(k))
        pos = rng.randrange(len(body) + 1)
        if rng.random() < 0.5:
            body = body[:pos] + "NEEDLE" + body[pos:]
        if rng.random() < 0.01:
            body += "é"
        rows.append("%s,%s" % (rng.choice("pq"), body))
    P = write_files(tmp_path, [["s.csv", "".join(r + "\n" for r in rows)]])
    for src in ["Dampr.text(P).filter(lambda l: 'NEEDLE' in l).count(lambda l: l.split(',')[0])",
                "Dampr.text(P).filter(lambda l: 'NEEDLE' not in l or l.endswith('NEEDLE')).count(lambda l: l.split(',')[0])",
                "Dampr.text(P).filter(lambda l: '' in l and l.startswith(('p,NEEDLE', 'q,'))).count(lambda l: l.split(',')[0])",
                "Dampr.text(P).filter(lambda l: 'é' in l or len(l) > 4000).count(lambda l: l.split(',')[0])",
                "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: 'EEDL' in r[1] and not r[1].endswith('z'))"
                ".count(lambda r: r[0])"]:
        check(src, P)


def test_undecided_leaves_on_both_sides(engine, tmp_path):
    rows = ["a,x", "b,x,1", "c,y,1,2,3,4,5,6,7,10", "d,y,1,2,3,4,5,6,7,-1", "e,y,q,2,3,4,5,6,7,zz"]
    P = write_files(tmp_path, [["u.csv", "".join(r + "\n" for r in rows * 400)]])
    src = "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: r[1] == 'x' or int(r[9]) > 0).count(lambda r: r[0])"
    with pytest.raises(ValueError):   # int('zz'): the device hands the e rows to the host, which raises
        run(src, P)
    P = write_files(tmp_path, [["v.csv", "".join(r + "\n" for r in rows[:4] * 400)]])
    check(src, P, host_lines=0, filtered=400)                    # r[9] is reached on the y rows only
    check("Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: r[0] == 'c' and int(r[9]) > 0 or r[1] == 'x')"
          ".count(lambda r: r[0])", P, host_lines=0, filtered=400)   # the U of r[9] behind a False is discarded
    check("Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: not (r[1] == 'y' and int(r[9]) < 0))"
          ".count(lambda r: r[0])", P, host_lines=0, filtered=400)


def test_nan_under_not(engine, tmp_path):
    """`not` is not a flipped comparison: NaN keeps the line (the device does not parse 'nan' and 'inf', so those
    lines are the host's, whose filter keeps them)"""
    P = write_files(tmp_path, [["n.csv", "a,1,2,nan\nb,1,2,0.5\nc,1,2,3.0\nd,1,2,inf\n" * 100]])
    check("Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: not (float(r[3]) < 1.0)).count(lambda r: r[0])",
          P, host_lines=200, filtered=100)


def random_program(rng, depth=0):
    """(source, leaves) of a random boolean program over the clean log's fields"""
    leaves = [
        "r[1] == 'GET'", "r[1] in ('PUT', 'POST')", "int(r[2]) >= 500", "float(r[4]) < 1.0", "len(r) == 7",
        "'ERROR' in r[5]", "'api' not in r[6]", "r[6].startswith(('/api', '/x'))", "r[6].endswith('.js')",
        "len(r[5]) > 2", "r[5].strip()", "int(r[9]) > 0", "r[0] < '3'", "len(r[6]) <= 2",
    ]
    if depth > 2 or rng.random() < 0.35:
        return rng.choice(leaves), 1
    if rng.random() < 0.2:
        s, n = random_program(rng, depth + 1)
        return "not (%s)" % s, n
    a, na = random_program(rng, depth + 1)
    b, nb = random_program(rng, depth + 1)
    return "(%s %s %s)" % (a, rng.choice(["and", "or"]), b), na + nb


def test_random_programs(engine, tmp_path):
    """programs of 1 .. 8 leaves against plain Python: results (exceptions included) and the device path"""
    text = "".join(l + "\n" for l in clean_log(5000, 6).split("\n")[1:-1] if not l.startswith("#"))
    P = write_files(tmp_path, [["r.csv", text]])
    rng = random.Random(7)
    done = 0
    while done < 40:
        prog, n = random_program(rng)
        if n > 8:
            continue
        src = "Dampr.text(P).map(lambda l: l.split(',')).filter(lambda r: %s).count(lambda r: r[1])" % prog
        try:
            exp = python_run(src, P)
        except IndexError:
            with pytest.raises(IndexError):
                run(src, P)
            done += 1
            continue
        got, (_s, how, d) = run(src, P)
        assert got == exp and NEEDLE in how, (src, d)
        done += 1


def test_json_string_tests_and_their_undecided_members(engine, tmp_path):
    """string tests on members: a string without escapes is decided on the device; an escaped string, a list or an
    object (where `in` and len() mean something else) is the host's, and so is a number, on which Python raises"""
    kinds = [{"k": "a", "m": "abc"}, {"k": "b", "m": " "}, {"k": "c", "m": ""}, {"k": "d", "m": "xyzw"},
             {"k": "e", "m": "a\"bc"}, {"k": "f", "m": "xé"}, {"k": "g", "m": ["abc", "x"]},
             {"k": "h", "m": {"abc": 1}}]
    recs = [kinds[i % len(kinds)] for i in range(4000)]
    P = write_files(tmp_path, [["j.jsonl", "".join(json.dumps(r) + "\n" for r in recs)]])
    # the escaped strings, the list and the object (2000 lines) go to the host; host_lines counts those its filter
    # keeps, filtered the lines the device drops
    check("Dampr.json(P).filter(lambda r: 'abc' in r['m'] or len(r['m']) > 3).count(lambda r: r['k'])", P,
          host_lines=1500, filtered=1000, detail=["sep=json"])   # kept: 'a"bc', the list, the object
    check("Dampr.json(P).filter(lambda r: not ('bc' not in r['m']) or len(r['m']) == 0).count(lambda r: r['k'])", P,
          host_lines=500, filtered=1000)                          # kept: 'a"bc'
    S = write_files(tmp_path, [["s.jsonl", "".join(json.dumps(r) + "\n" for r in recs if isinstance(r["m"], str))]])
    check("Dampr.json(P).filter(lambda r: r['m'].strip() and not r['m'].endswith('c') or r['m'].startswith(('a', 'x')))"
          ".count(lambda r: r['k'])", S, host_lines=1000, filtered=1000)
    N = write_files(tmp_path, [["n.jsonl", "".join(json.dumps(r) + "\n" for r in recs[:8] + [{"k": "z", "m": 7}])]])
    with pytest.raises(AttributeError):
        run("Dampr.json(P).filter(lambda r: r['m'].startswith(('a', 'x'))).count(lambda r: r['k'])", N)
    with pytest.raises(TypeError):
        run("Dampr.json(P).filter(lambda r: r['k'] == 'a' or len(r['m']) > 1).count(lambda r: r['k'])", N)
