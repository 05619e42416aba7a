"""Random filter programs over the fuzzed corpora of tests/fields_fuzz.py (imported, not changed), and the per-line
outcome of each: TAKE (every filter holds), DROP (one is false) or HOST (the device cannot decide, or Python raises).
Shared by test_fields_filter_fuzz.py (the stand-in of tests/fields_filter_standin.py against CPython) and
test_gpu_fields_filter_fuzz.py (the kernels against both).

A stage is `Dampr.text(P)[.filter(LINE)].map(split)[.filter(FIELDS)].mean(lambda r: 1, lambda r: 1)`: a constant key
and value, so a line the filters keep is always taken and its outcome is the filters' verdict alone. LINE is a program
over the whole line, FIELDS one over the split record; together they hold 1 .. 8 leaves joined by and / or / not.
The leaves are the single predicates of fields_fuzz.text_filter and the string tests (substring, prefix, suffix,
length, non-blank, whole-line comparisons), with needles that are empty, non-ASCII or longer than most fields."""
import random

import fields_fuzz as fz
from fields_filter_standin import line_verdict

TAKE, DROP, HOST = fz.TAKE, fz.DROP, fz.HOST
NEEDLES = ["", "a", "ab", "x", "0", "-", ".", "7", "AB_", "é", "abcxyzAB_-.07abc", "\t"]


def _needle(rng):
    return repr(rng.choice(NEEDLES))


def field_leaf(rng):
    if rng.random() < 0.4:
        return fz.text_filter(rng)
    i = fz._idx(rng, "s")
    return rng.choice([
        "%s in r[%d]" % (_needle(rng), i), "%s not in r[%d]" % (_needle(rng), i),
        "r[%d].startswith(%s)" % (i, _needle(rng)), "r[%d].endswith((%s, %s))" % (i, _needle(rng), _needle(rng)),
        "len(r[%d]) %s %d" % (i, rng.choice(fz.CMPS), rng.randrange(6)), "r[%d].strip()" % i])


def line_leaf(rng):
    return rng.choice([
        "%s in l" % _needle(rng), "%s not in l" % _needle(rng), "l.startswith((%s, %s))" % (_needle(rng), _needle(rng)),
        "l.endswith(%s)" % _needle(rng), "len(l) %s %d" % (rng.choice(fz.CMPS), rng.choice([0, 1, 10, 40, 4095])),
        "l.strip()", "l != ''", "l %s %s" % (rng.choice(fz.CMPS), _needle(rng)), "l in ('', 'a', ' ')"])


def program(rng, leaf, n):
    """the source of a random and / or / not tree over n leaves"""
    if n == 1:
        s = leaf(rng)
    else:
        k = rng.randint(1, n - 1)
        s = "(%s %s %s)" % (program(rng, leaf, k), rng.choice(["and", "or"]), program(rng, leaf, n - k))
    return "not (%s)" % s if rng.random() < 0.15 else s


class Stage(object):
    """a generated stage: its lambdas, source and (after match) the device predicates and call"""

    def __init__(self, rng, family):
        self.family = family
        n = rng.randint(1, 8)
        nl = rng.randint(0, min(n, 3)) if rng.random() < 0.6 else 0
        self.line_src = program(rng, line_leaf, nl) if nl else None
        self.field_src = program(rng, field_leaf, n - nl) if n > nl else None
        split = "l.split(',')" if family == "sep" else "l.split()"
        self.src = "Dampr.text(P)" + (".filter(lambda l: %s)" % self.line_src if self.line_src else "") + \
            ".map(lambda l: %s)" % split + (".filter(lambda r: %s)" % self.field_src if self.field_src else "") + \
            ".mean(lambda r: 1, lambda r: 1)"
        self.line_fn = eval("lambda l: " + self.line_src) if self.line_src else None
        self.field_fn = eval("lambda r: " + self.field_src) if self.field_src else None
        self.split = (lambda l: l.split(",")) if family == "sep" else (lambda l: l.split())

    def match(self, path):
        """the planner's (spec, op, expr, preds) of the stage over the text file `path`, or None"""
        from dampr_b200 import Dampr, plan
        pm = eval(self.src, {"Dampr": Dampr, "P": path})
        st = pm.pmer.graph.stages[0]
        m = plan._match_text_fields(st, [pm.pmer.graph.inputs[st.inputs[0]]], programs=True)
        if m is None:
            return None
        _src, spec, op, _mean, preds, expr = m
        self.spec, self.op, self.expr, self.preds = spec, op, expr, preds
        return m


def python_outcome(stage, line):
    """CPython's outcome of one line (bytes): the stage's own filters, HOST when one raises"""
    s = line.decode("utf-8")
    try:
        if stage.line_fn is not None and not stage.line_fn(s):
            return DROP
        return TAKE if stage.field_fn is None or stage.field_fn(stage.split(s)) else DROP
    except Exception:
        return HOST


def fields_of(family, line):
    """the split record as bytes fields (str.split() for the whitespace family, on the decoded line)"""
    if family == "sep":
        return line.split(b",")
    return [x.encode("utf-8") for x in line.decode("utf-8").split()]


def standin_outcome(stage, line, cr):
    v = line_verdict(line, fields_of(stage.family, line), stage.preds, cr)
    return HOST if v is None else TAKE if v else DROP


def corpus_lines(family, seed, n, cr):
    data = fz.corpus(family, seed, n, cr)
    return data, fz.lines_of(data)


def stages(seed, family, count, path):
    """count generated stages that the planner lowers, and how many it refused on the way"""
    rng = random.Random(seed)
    out, refused = [], 0
    while len(out) < count:
        st = Stage(rng, family)
        if st.match(path) is None:
            refused += 1
            continue
        out.append(st)
    return out, refused
