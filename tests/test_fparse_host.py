"""parse_f64 (dampr_b200/csrc/fparse.cuh), compiled as host code, against Python's float() on a seeded corpus of
more than 2 * 10^6 strings; and the committed power-of-five table against its generator (tools/gen_pow5.py).

The parser is the device's float() of the field scan: every string it accepts must give float()'s bits, and it may
refuse only what its grammar leaves out, or a string whose rounding the truncated table cannot decide (counted, and
bounded). A small shared object is built from the header into tmp_path with nvcc, so the product library carries
no test hook; the test skips where nvcc is absent."""
import ctypes as C
import importlib.util
import os
import random
import re
import shutil
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dampr_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"

SHIM = r"""
#include "fparse.cuh"
extern "C" void fp_parse_many(const unsigned char *buf, const unsigned long long *offs, unsigned long long n,
                              double *out, unsigned char *ok) {
    for (unsigned long long i = 0; i < n; ++i) {
        double d = 0.0;
        ok[i] = parse_f64(buf + offs[i], (uint32_t)(offs[i + 1] - offs[i]), d) ? 1 : 0;
        out[i] = d;
    }
}
"""

# the grammar the parser takes: surrounding ' ' / '\t', [+-]?(\d+\.?\d*|\.\d+)([eE][+-]?\d+)?
GRAMMAR = re.compile(r"[ \t]*[+-]?([0-9]+\.?[0-9]*|\.[0-9]+)([eE][+-]?[0-9]+)?[ \t]*\Z")


def in_grammar(s):
    """the parser must accept s (unless the table cannot decide its rounding)"""
    m = GRAMMAR.match(s)
    if not m:
        return False
    digits = m.group(1).replace(".", "").lstrip("0")
    return len(digits) <= 19


@pytest.fixture(scope="module")
def parse(tmp_path_factory):
    if not os.path.exists(NVCC) and not shutil.which(NVCC):
        pytest.skip("nvcc not available")
    d = tmp_path_factory.mktemp("fparse")
    src, lib = os.path.join(str(d), "shim.cu"), os.path.join(str(d), "shim.so")
    with open(src, "w") as f:
        f.write(SHIM)
    subprocess.check_call([NVCC, "-x", "cu", "-shared", "-Xcompiler", "-fPIC", "-O2", "-std=c++17",
                           "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC, src, "-o", lib])
    so = C.CDLL(lib)
    so.fp_parse_many.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    so.fp_parse_many.restype = None

    def run(strs):
        bs = [s.encode("utf-8") for s in strs]
        buf = np.frombuffer(b"".join(bs) + b"\0", dtype=np.uint8)
        offs = np.zeros(len(bs) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(b) for b in bs])
        out = np.zeros(len(bs), dtype=np.float64)
        ok = np.zeros(len(bs), dtype=np.uint8)
        so.fp_parse_many(buf.ctypes.data, offs.ctypes.data, len(bs), out.ctypes.data, ok.ctypes.data)
        return out, ok.astype(bool)
    return run


def f64(bits):
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def random_double(rng):
    """every binade, subnormals included, both signs"""
    return f64((rng.getrandbits(1) << 63) | (rng.randrange(0, 2047) << 52) | rng.getrandbits(52))


BOUNDARIES = ["2.4703282292062327e-324", "2.4703282292062328e-324", "4.9406564584124654e-324",
              "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308",
              "2.2250738585072011e-308", "2.2250738585072014e-308", "2.2250738585072012e-308",
              "9007199254740993", "9007199254740992", "9007199254740994", "9007199254740995", "9007199254740997",
              "18014398509481987", "18014398509481989", "1e23", "8.589973e9", "1e22", "1e-22", "4.35e-5"]
SPELLINGS = ["0", "-0", "+0", "0.0", "-0.0", "00.00e5", ".5", "5.", "-.5", "+5.", "007", "5e0", "5E+0", "5e-0",
             "5e0000000000000000000000001", "1e999999", "-1e999999", "0e999999", "-0e999999", "1e-999999",
             "-1e-999", "1e308", "1e309", "0.1e309", "1e-324", "3e-324", " 1.5", "1.5 ", "\t-2.5e3\t", "  7  ",
             "1234567890123456789", "12345678901234567890", "1.234567890123456789", "0.0000000000000000000001",
             "1000000000000000000000", "100000000000000000000e-3", "1.0000000000000000000",
             "000000000000000000000000001.5"]
REJECTED = ["inf", "-inf", "Infinity", "nan", "NaN", "-nan", "iNfInItY", "1_0.5", "1_000", "1.5\v", "1.5\f",
            "\x1c1.5", "1.5\n", "", " ", "\t", "1e", "1e+", ".", "-.", "e5", "--1", "+-1", "1.2.3", "1e5.5", "0x10",
            "1,5", "１", "1.5e", "1 .5", "1. 5", "- 1"]


def corpus(seed=20261015):
    """(kind, string) pairs, over 2 * 10^6 of them"""
    rng = random.Random(seed)
    out = []
    for _ in range(600000):
        out.append(("repr", repr(random_double(rng))))
    for _ in range(1300000):
        d = random_double(rng) if rng.random() < 0.7 else rng.uniform(-1e6, 1e6)
        fmt = "%%.%d%s" % (rng.randrange(0, 19), rng.choice("efg"))
        s = fmt % d
        if len(s) < 400:
            out.append(("fmt", s))
    for _ in range(100000):   # exact halfway integers above 2^53: ties to even, both ways
        k = rng.randrange(53, 63)
        out.append(("tie", str((1 << k) + (2 * rng.randrange(0, 1 << (k - 53)) + 1) * (1 << (k - 53)))))
    for _ in range(100000):   # 19- and 20-digit mantissas, with a point and an exponent
        nd = rng.choice((18, 19, 19, 20, 21))
        m = str(rng.randrange(10 ** (nd - 1), 10 ** nd))
        p = rng.randrange(0, nd + 1)
        out.append(("digits", "%s%s.%se%d" % (rng.choice(("", "-")), m[:p], m[p:], rng.randrange(-330, 310))))
    for _ in range(50000):    # leading / trailing zeros, signs, exponent spellings
        m = "%d" % rng.randrange(1, 10 ** rng.randrange(1, 17))
        s = "0" * rng.randrange(0, 4) + m[:1] + "." + m[1:] + "0" * rng.randrange(0, 4)
        s = rng.choice(("", "+", "-")) + s + rng.choice(("", "e%d" % rng.randrange(-40, 40),
                                                          "E+%03d" % rng.randrange(0, 300), "e-%d" % rng.randrange(0, 330)))
        out.append(("spell", s))
    out += [("fixed", s) for s in BOUNDARIES + SPELLINGS + REJECTED]
    return out


def test_parse_f64_matches_python_float(parse):
    cases = corpus()
    assert len(cases) >= 2000000
    strs = [s for _k, s in cases]
    got, ok = parse(strs)
    wrong, outside, undecided, refused_repr = [], [], [], 0
    n_repr = 0
    for (kind, s), g, k in zip(cases, got.tolist(), ok.tolist()):
        n_repr += kind == "repr"
        must = in_grammar(s)
        if k:
            if not must:
                outside.append(s)          # accepted a string outside the grammar
                continue
            if struct.pack("<d", g) != struct.pack("<d", float(s)):
                wrong.append((s, g, float(s)))
        elif must:
            undecided.append(s)
            refused_repr += kind == "repr"
    print("parse_f64: %d strings, %d repr strings refused (of %d), %d refused in total within the grammar"
          % (len(cases), refused_repr, n_repr, len(undecided)))
    assert not wrong, wrong[:10]
    assert not outside, outside[:10]
    assert refused_repr * 10 ** 6 <= 10 * n_repr, undecided[:10]
    assert len(undecided) * 10 ** 6 <= 10 * len(cases), undecided[:10]


def test_parse_f64_fixed_cases(parse):
    """the boundaries, ties and spellings one by one, with the values Python gives"""
    strs = BOUNDARIES + SPELLINGS + REJECTED
    got, ok = parse(strs)
    res = dict(zip(strs, zip(got.tolist(), ok.tolist())))
    for s in BOUNDARIES + SPELLINGS:
        if in_grammar(s):
            v, k = res[s]
            assert k and struct.pack("<d", v) == struct.pack("<d", float(s)), (s, v, float(s))
        else:
            assert not res[s][1], s
    for s in REJECTED:
        assert not res[s][1], s
    assert res["9007199254740993"][0] == 9007199254740992.0     # a tie rounds to even: down ...
    assert res["9007199254740995"][0] == 9007199254740996.0     # ... and up
    assert res["1e999999"][0] == float("inf") and res["-1e999999"][0] == float("-inf")
    assert struct.pack("<d", res["-1e-999"][0]) == struct.pack("<d", -0.0)
    assert not res["12345678901234567890"][1] and not res["1.0000000000000000000"][1]   # 20 significant digits
    assert res["1234567890123456789"][1] and res["000000000000000000000000001.5"][1]


def test_pow5_header_matches_its_generator():
    spec = importlib.util.spec_from_file_location("gen_pow5", os.path.join(ROOT, "tools", "gen_pow5.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    with open(os.path.join(CSRC, "pow5.cuh")) as f:
        assert f.read() == gen.render()
    # spot checks of the definition: 5^0 scaled to bit 127, and 5^-1 rounded up
    assert gen.entry(0) == 1 << 127
    assert gen.entry(-1) == (1 << 130) // 5 + 1
    assert all((1 << 127) <= gen.entry(q) < (1 << 128) for q in range(gen.Q_MIN, gen.Q_MAX + 1))
