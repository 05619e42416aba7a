"""CPU: a plain-Python statement of the 64-bit key codes the text and field kernels give tokens and keys, and the
pairs of different long tokens in tests/golden/code_collisions.json (tools/find_code_collisions.py) that share one.

Tokens longer than an exact code holds (12 symbols in the [^\\w]+ modes, 9 bytes for str.split and field keys, and
the field key '') are hashed: csrc/text2.cu token_code2, csrc/text.cu token_code and csrc/fields.cu hash_bytes all
compute 1 << 63 | mix64((h1 << 32 | h2) ^ len * 0x9E3779B97F4A7C15) under the fixed seed 0x243F6A8885A308D3. The
engine's answers equal Python's only because every kernel byte-compares the tokens that share a code (DAMPR_TF_COLLISION
sends the stage to the host map); tests/test_gpu_code_collisions.py runs the kernels on these pairs. Here: the pairs
collide under the statement, in the way that lets the GPU tests extend and re-case them, and the statement draws the
exact/hashed boundary where the host decoder (dampr_b200/keycodes.py) expects it. Also the host side of the same
guard: HASH-class Python keys whose 64-bit codes collide (keycodec) still fold, join and de-duplicate like Python."""
import collections
import json
import os
import random

import numpy as np
import pytest

from dampr_b200 import keycodes
from dampr_b200 import device as dev

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "code_collisions.json")

SEED = 0x243F6A8885A308D3
M32, M64 = (1 << 32) - 1, (1 << 64) - 1
MAXEXACT = {"raw": 9, "sym": 12}
SYM = {c: i + 1 for i, c in enumerate(b"0123456789_abcdefghijklmnopqrstuvwxyz")}   # '0' -> 1 .. 'z' -> 37


def mix64(x):
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & M64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def symbol(c):
    """[^\\w]+ modes: the symbol of an ASCII word byte, letters case-folded"""
    return SYM[c | 0x20 if 0x41 <= c <= 0x5A else c]


def hash_state(token, variant):
    """(h1 << 32 | h2) of the kernels' two running hashes after the bytes of token"""
    h1, h2 = (SEED & M32) ^ 0x811C9DC5, (SEED >> 32) ^ 0x9747B28C
    for c in token:
        v = symbol(c) if variant == "sym" else c
        h1 = ((h1 ^ v) * 16777619) & M32
        h2 = ((h2 ^ v) * 0x85EBCA6B + 0x9E3779B9) & M32
        h2 = ((h2 << 13) | (h2 >> 19)) & M32
    return (h1 << 32) | h2


def long_code(token, variant):
    """the hashed code of token (bytes): variant 'raw' (str.split tokens, field keys) or 'sym' ([^\\w]+ tokens)"""
    return mix64(hash_state(token, variant) ^ ((len(token) * 0x9E3779B97F4A7C15) & M64)) | (1 << 63)


def key_code(token, variant, field_key=False):
    """the code a kernel gives token: exact packing when it fits (7 bits per byte, first byte lowest; base 38 per
    symbol, first symbol lowest), the hashed code otherwise. str.split tokens with a NUL and the field key '' hash."""
    if len(token) <= MAXEXACT[variant] and not (variant == "raw" and (0 in token or (field_key and not token))):
        code = 0
        for c in reversed(token):
            code = code * 38 + symbol(c) if variant == "sym" else (code << 7) | c
        return code
    return long_code(token, variant)


def load_pairs():
    with open(GOLDEN) as f:
        doc = json.load(f)
    return {v: [(p["a"].encode(), p["b"].encode(), int(p["state"], 16), int(p["code"], 16)) for p in pairs]
            for v, pairs in doc["variants"].items()}


PAIRS = load_pairs()


@pytest.mark.parametrize("variant", ["raw", "sym"])
def test_every_fixture_pair_collides_at_the_state(variant):
    assert len(PAIRS[variant]) >= 3
    for a, b, state, code in PAIRS[variant]:
        assert a != b and a.lower() != b.lower() and len(a) == len(b) > MAXEXACT[variant]
        assert all(c in b"abcdefghijklmnopqrstuvwxyz0123456789" for c in a + b)   # word characters, no separators
        assert hash_state(a, variant) == hash_state(b, variant) == state
        assert long_code(a, variant) == long_code(b, variant) == code
        assert key_code(a, variant) == code and code >> 63
    other = {"raw": "sym", "sym": "raw"}[variant]
    for a, b, _s, _c in PAIRS[variant]:
        assert long_code(a, other) != long_code(b, other)   # a pair is a pair of one variant only


@pytest.mark.parametrize("variant", ["raw", "sym"])
def test_suffix_extended_pairs_still_collide(variant):
    rng = random.Random(variant)
    for a, b, _s, _c in PAIRS[variant]:
        for n in (1, 2, 19, 20, 31, 4000):
            s = bytes(rng.choice(b"abcdefghijklmnopqrstuvwxyz0123456789_") for _ in range(n))
            assert long_code(a + s, variant) == long_code(b + s, variant)
            assert long_code(a + s, variant) != long_code(a, variant)
        assert long_code(b"x" + a, variant) != long_code(b"x" + b, variant)   # a common prefix does not keep it


def test_case_variants_collide_in_sym_mode_only():
    rng = random.Random(7)
    for a, b, _s, code in PAIRS["sym"]:
        for _ in range(8):
            ua = bytes(c - 32 if 0x61 <= c <= 0x7A and rng.random() < 0.5 else c for c in a)
            ub = b.upper()
            assert long_code(ua, "sym") == long_code(ub, "sym") == code
            if ua != a:
                assert long_code(ua, "raw") != long_code(a, "raw")


@pytest.mark.parametrize("variant,mode", [("sym", dev.TOK_NONWORD_LOWER), ("raw", dev.TOK_WS)])
def test_exact_hashed_boundary(variant, mode):
    """12 symbols / 9 bytes get an exact code below 2^63 that the host decoder turns back into the token; one more
    symbol or byte gets a hashed code (bit 63 set); the field key '' and a str.split token with a NUL hash too"""
    m = MAXEXACT[variant]
    rng = random.Random(m)
    alpha = b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_"
    for n in range(1, m + 2):
        for tok in (bytes(rng.choice(alpha) for _ in range(n)), b"z" * n, b"_" * n, b"Z" * n, b"9" * n):
            code = key_code(tok, variant)
            if n <= m:
                assert code < 1 << 63
                want = tok.decode() if variant == "raw" else tok.decode().lower()
                assert keycodes.decode_exact(np.array([code], np.uint64), mode) == [want]
            else:
                assert code >> 63 and code == long_code(tok, variant)
    assert key_code(b"z" * 9, "raw") == sum(0x7A << (7 * i) for i in range(9))
    assert key_code(b"z" * 12, "sym") == 38 ** 12 - 1 < 1 << 63 < 38 ** 13
    assert key_code(b"", "raw", field_key=True) == long_code(b"", "raw")
    assert key_code(b"a\0", "raw") >> 63


# ---- the host side: HASH-class Python keys with colliding 64-bit codes ---------------------------------------------
@pytest.fixture
def two_bit_hash(monkeypatch):
    """every HASH-class key gets one of four codes, so almost every pair of distinct keys collides"""
    from dampr_b200 import keycodec, settings
    from dampr_b200 import runner as runner_mod
    from fake_device import FakeCtx
    monkeypatch.setattr(runner_mod, "_CTX", {settings.device: FakeCtx()})
    orig = keycodec._hash_code
    monkeypatch.setattr(keycodec, "_hash_code", lambda k: orig(k) & 3)
    yield


def hash_keys(rng, n):
    pool = [None, (1, "a"), (1, "b"), ("a", 1), (2,), (), ("x", None), (1.5, 2), ("é", ("n", 3)), frozenset([1, 2]),
            (True, 0), (1, 0), (0, 1), ("", ""), ((),), (None, None)]
    return [rng.choice(pool) for _ in range(n)]


def test_hash_keys_fold_by_key_under_colliding_codes(two_bit_hash):
    from dampr_b200 import Dampr
    rng = random.Random(11)
    rows = [(k, rng.randrange(-50, 50)) for k in hash_keys(rng, 4000)]
    got = dict(Dampr.memory(rows).a_group_by(lambda r: r[0], lambda r: r[1]).sum().read())
    exp = collections.defaultdict(int)
    for k, v in rows:
        exp[k] += v
    assert got == dict(exp)
    got = dict(Dampr.memory(rows).group_by(lambda r: r[0], lambda r: r[1]).reduce(lambda k, it: sorted(it)).read())
    exp = collections.defaultdict(list)
    for k, v in rows:
        exp[k].append(v)
    assert got == {k: sorted(v) for k, v in exp.items()}
    got = dict(Dampr.memory(rows).group_by(lambda r: r[0], lambda r: r[1] % 5).unique().read())
    exp = {}
    for k, v in rows:
        seen = exp.setdefault(k, [])
        if v % 5 not in seen:
            seen.append(v % 5)
    assert {k: sorted(v) for k, v in got.items()} == {k: sorted(v) for k, v in exp.items()}


def test_hash_keys_join_under_colliding_codes(two_bit_hash):
    from dampr_b200 import Dampr
    rng = random.Random(12)
    left = [(k, rng.randrange(100)) for k in hash_keys(rng, 600)]
    right = [(k, rng.randrange(100)) for k in hash_keys(rng, 500)[:-100]]
    L = Dampr.memory(left).group_by(lambda r: r[0], lambda r: r[1])
    R = Dampr.memory(right).group_by(lambda r: r[0], lambda r: r[1])
    got = dict(L.join(R).reduce(lambda l, r: (sorted(l), sorted(r))).read())
    lg, rg = collections.defaultdict(list), collections.defaultdict(list)
    for k, v in left:
        lg[k].append(v)
    for k, v in right:
        rg[k].append(v)
    assert got == {k: (sorted(lg[k]), sorted(rg[k])) for k in lg if k in rg}
    got = dict(L.join(R).left_reduce(lambda l, r: (sum(l), sum(r))).read())
    assert got == {k: (sum(lg[k]), sum(rg.get(k, ()))) for k in lg}
