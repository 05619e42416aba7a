"""Seeded corpora that sit on the text kernels' structural seams, and a plain-Python statement of the C-ABI contract
(include/dampr_b200.h: dampr_text_count, dampr_table_fallback_lines, dampr_text_fields) they are checked against.

No native library is needed here: the CPU suite checks the generators reach their seams and that the contract
oracle composes back to the reference semantics (oracle/refsem.py); the GPU suite runs the kernels on the same
corpora. Every offset is a byte offset into the corpus, relative to own_lo = 0 of a whole-range call.

The kernel constants restated here (a change to one of them must be mirrored, or the coverage tests stop meaning
what they say):
  csrc/text2.cu:36-43   V_STRIP = 2048, V_OWN = 16384, V_LEAD = 32, V_WIN = 18464, V_HCAP = 256
  csrc/text2.cu:85      HCAP = 256, 128, 64 for the 2-, 3- and 4-CTA builds
  csrc/text2.cu:63      V_MAXBAD = 8 host lines per warp region (the lines that start in one strip)
  csrc/text2.cu:217     exact key codes: 9 bytes (str.split), 12 symbols ([^\\w]+)
  csrc/text.cu:34-37    first-generation kernel: T_LEAD = 32, T_OWN = 6144, T_WIN = 10272
  csrc/fields.cu:31-36  F_OWN = 16384, F_HALO = 4096 (longest device line, '\\n' included), F_FB_MAXLEN = 65535
"""
import bisect
import random
import re

TOK_WS, TOK_NONWORD_LOWER_SET, TOK_NONWORD_LOWER = 0, 1, 2          # include/dampr_b200.h:126-128
TF_NONASCII, TF_CR, TF_LONGLINE, TF_TABLEFULL, TF_LONGTOKEN, TF_COLLISION = 1, 2, 4, 8, 16, 32
FIELD_KEY_STR, FIELD_KEY_INT, FIELD_VAL_ONE = 0, 1, 0x7FFFFFFF
OP_SUM_I64, OP_MIN_I64, OP_MAX_I64 = 0, 3, 4

V_STRIP = 2048
V_OWN = 16384
V_LEAD = 32
V_WIN = 18464
V_WIN_END = V_WIN - V_LEAD            # a line owned by a tile must end (its '\n') before tile start + 18432
HCAP = {4: 64, 3: 128, 2: 256}
V_MAXBAD = 8
T_OWN = 6144
T_WIN_END = 10272 - 32
F_OWN = 16384
F_HALO = 4096
F_FB_MAXLEN = 0xFFFF

RX = re.compile(r"[^\w]+")            # benchmarks/tf-idf-dampr.py:11
WS_BYTES = b"\t\n\x0b\x0c\r\x1c\x1d\x1e\x1f "   # str.split() whitespace within ASCII
WS_TOKEN = re.compile(rb"[^\t\n\x0b\x0c\r\x1c-\x20]+")
WORD = b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_"


# ---- lines as the kernels see them ---------------------------------------------------------------------------------
def nl_lines(data):
    """(offset, length) of every line split at '\\n' only; a last line without '\\n' is a line, text after the final
    '\\n' is not. These are the kernels' lines: a line starts at 0 or after a '\\n', below n."""
    out, pos, n = [], 0, len(data)
    while pos < n:
        e = data.find(b"\n", pos)
        e = n if e < 0 else e
        out.append((pos, e - pos))
        pos = e + 1
    return out


def text_mode_lines(b):
    """the lines Python's text mode makes of bytes b (universal newlines), as str"""
    s = b.decode("utf-8").replace("\r\n", "\n").replace("\r", "\n")
    parts = s.split("\n")
    if parts and parts[-1] == "":
        parts.pop()
    return parts


def python_lines(b, cr_is_data):
    """lines of bytes b as the reference reads them: binary-mode .gz splits at '\\n' only, text mode also at '\\r'"""
    if cr_is_data:
        return [b[o:o + ln].decode("utf-8") for o, ln in nl_lines(b)]
    return text_mode_lines(b)


def host_lines(line, cr_is_data):
    """the reference's lines (str) of one '\\n' line of the text, which the device handed back"""
    return python_lines(line + b"\n", cr_is_data)


def line_is_bad(line, cr_is_data):
    """a line the [^\\w]+ tokenisers hand to the host (dampr_b200.h:158-165): a non-ASCII byte, or '\\r' in text mode"""
    return any(c >= 0x80 for c in line) or (not cr_is_data and b"\r" in line)


def python_tokens(line_str, mode):
    if mode == TOK_WS:
        return line_str.split()
    toks = RX.split(line_str.lower())
    return set(toks) if mode == TOK_NONWORD_LOWER_SET else toks


# ---- dampr_text_count ------------------------------------------------------------------------------------------------
def expected_fallback(data, kernel, mode, cr_is_data):
    """the exact (offset << 16) | length entries dampr_table_fallback_lines reports when no refusal flag is set:
    only the second-generation kernel hands lines back, and only in the [^\\w]+ modes"""
    if kernel != 2 or mode == TOK_WS:
        return []
    return sorted((o << 16) | ln for o, ln in nl_lines(data) if line_is_bad(data[o:o + ln], cr_is_data))


def expected_table(data, mode, cr_is_data, fallback=()):
    """{token: count} over the lines not in `fallback`, plus the counters dampr_table_stats reports:
    lines (the '\\n' lines counted on the device), empty (the '' token), folded (tokens folded, '' excluded)"""
    skip = {int(e) >> 16 for e in fallback}
    table, lines, empty, folded = {}, 0, 0, 0
    for o, ln in nl_lines(data):
        if o in skip:
            continue
        lines += 1
        toks = python_tokens(data[o:o + ln].decode("ascii"), mode)
        for t in toks:
            if t == "":
                empty += 1
                continue
            folded += 1
            table[t] = table.get(t, 0) + 1
    return {"table": table, "lines": lines, "empty": empty, "folded": folded}


def python_over_lines(data, offsets, mode, cr_is_data):
    """{token: count} and the '' count of the reference run over the given '\\n' lines only (the host's share)"""
    table, empty, nlines = {}, 0, 0
    starts = set(offsets)
    for o, ln in nl_lines(data):
        if o not in starts:
            continue
        for l in host_lines(data[o:o + ln], cr_is_data):
            nlines += 1
            for t in python_tokens(l, mode):
                if t == "":
                    empty += 1
                else:
                    table[t] = table.get(t, 0) + 1
    return table, empty, nlines


def distinct_tokens(line, mode=TOK_NONWORD_LOWER_SET):
    return len(set(RX.split(line.decode("ascii").lower())) - {""})


def refusals(data, mode, cr_is_data, ranges, kernel, ctas=4):
    """(required, allowed) flag masks of dampr_text_count over the ownership ranges `ranges`.
    required: the flags the kernel must set; allowed: the flags it may set. When required holds a refusal flag the
    scan is the caller's and the table carries no promise; when allowed is 0 the table must be exact."""
    n = len(data)
    nonascii = any(c >= 0x80 for c in data)
    has_cr = b"\r" in data
    if mode == TOK_WS:
        req = (TF_NONASCII if nonascii else 0) | (TF_CR if has_cr and (kernel == 1 or not cr_is_data) else 0)
        return req, req
    lines = nl_lines(data)
    starts = [o for o, _ in lines]
    end_of = dict((o, o + ln) for o, ln in lines)   # position of the '\n' (n reads as '\n')
    if kernel == 1:
        req = (TF_NONASCII if nonascii else 0) | (TF_CR if has_cr else 0)
        own, strip, win_end = T_OWN, T_OWN, T_WIN_END
    else:
        req = 0
        own, strip, win_end = V_OWN, V_STRIP, V_WIN_END
    allowed = 0
    for lo, hi in ranges:
        for t0 in range(lo, hi, own):
            for s0 in range(t0, min(t0 + own, hi), strip):
                s1 = min(s0 + strip, hi)
                a, b = bisect.bisect_left(starts, s0), bisect.bisect_left(starts, s1)
                if a == b:
                    continue
                if end_of[starts[b - 1]] >= t0 + win_end:
                    req |= TF_LONGLINE        # the region's last line does not end inside the window
                    continue
                if kernel == 2:
                    nbad = sum(1 for x in starts[a:b] if line_is_bad(data[x:end_of[x]], cr_is_data))
                    if nbad > V_MAXBAD:
                        req |= TF_NONASCII
                    if mode == TOK_NONWORD_LOWER_SET:
                        for x in starts[a:b]:
                            l = data[x:end_of[x]]
                            if not line_is_bad(l, cr_is_data) and distinct_tokens(l) > HCAP[ctas]:
                                allowed |= TF_LONGLINE   # more distinct tokens than the set() history holds
    return req, req | allowed


# ---- dampr_text_fields -----------------------------------------------------------------------------------------------
INT18 = re.compile(rb"[+-]?[0-9]{1,18}")


def _field(f, i):
    return f[i] if -len(f) <= i < len(f) else None


def field_line_to_host(line, spec, cr_is_data):
    """True when the device hands this '\\n' line to the host (dampr_b200.h:182-191)"""
    sep, kf, kind, vf, _op = spec
    if len(line) >= F_HALO or any(c >= 0x80 or c == 0 for c in line) or (not cr_is_data and b"\r" in line):
        return True
    f = line.split(bytes([sep]))
    k = _field(f, kf)
    v = f[0] if vf == FIELD_VAL_ONE else _field(f, vf)
    if k is None or v is None:
        return True
    if vf != FIELD_VAL_ONE and not INT18.fullmatch(v):
        return True
    return kind == FIELD_KEY_INT and not INT18.fullmatch(k)


def fields_prediction(data, spec, cr_is_data):
    """what dampr_text_fields must report over the whole text (any ownership split):
    flags (TF_LONGLINE iff a line is 65536 bytes or longer), the exact fallback list, and the fold over the other
    lines: {key: value} (str keys, or int keys for FIELD_KEY_INT), lines, folded, max_abs"""
    sep, kf, kind, vf, op = spec
    flags, fb, acc, nlines, max_abs = 0, [], {}, 0, 0
    for o, ln in nl_lines(data):
        line = data[o:o + ln]
        if field_line_to_host(line, spec, cr_is_data):
            if ln > F_FB_MAXLEN:
                flags |= TF_LONGLINE
            else:
                fb.append((o << 16) | ln)
            continue
        f = line.split(bytes([sep]))
        key = f[kf].decode("ascii")
        if kind == FIELD_KEY_INT:
            key = int(key)
        v = 1 if vf == FIELD_VAL_ONE else int(f[vf])
        nlines += 1
        max_abs = max(max_abs, abs(v))
        acc[key] = fold(op, acc[key], v) if key in acc else v
    if op == OP_SUM_I64:
        acc = {k: wrap64(v) for k, v in acc.items()}
    return {"flags": flags, "fallback": sorted(fb), "table": acc, "lines": nlines, "folded": nlines,
            "max_abs": max_abs}


def fold(op, a, b):
    return a + b if op == OP_SUM_I64 else (min(a, b) if op == OP_MIN_I64 else max(a, b))


def wrap64(v):
    """two's-complement int64 of v: the device's SUM"""
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >> 63 else v


ERR = "\0error"


def field_functions(spec):
    """the stage's own functions, l.split(S)[i] / int(l.split(S)[j]), with a raised exception mapped to ERR / 0 so
    that whole-text runs over lines Python refuses can still be compared"""
    sep, kf, kind, vf, _op = spec
    s = chr(sep)

    def key(l):
        try:
            return int(l.split(s)[kf]) if kind == FIELD_KEY_INT else l.split(s)[kf]
        except (IndexError, ValueError):
            return ERR

    def value(l):
        if vf == FIELD_VAL_ONE:
            return 1
        try:
            return int(l.split(s)[vf])
        except (IndexError, ValueError):
            return 0
    return key, value


def python_fold_lines(lines, spec):
    key, value = field_functions(spec)
    out = {}
    for l in lines:
        k, v = key(l), value(l)
        out[k] = fold(spec[4], out[k], v) if k in out else v
    return out


# ---- corpora ---------------------------------------------------------------------------------------------------------
class Writer(object):
    """appends lines; no line may start exactly on a strip seam, so a line straddles every 2 KB seam it meets"""

    def __init__(self, rng):
        self.rng = rng
        self.buf = bytearray()

    def line(self, body):
        if (len(self.buf) + len(body) + 1) % V_STRIP == 0:
            body = body + b" "
        self.buf += body + b"\n"

    def filler_line(self, maxlen=80):
        r = self.rng
        words = [bytes(r.choice(WORD) for _ in range(r.randint(1, 7))) for _ in range(r.randint(1, maxlen // 8))]
        self.line(b" ".join(words))

    def pad_to(self, target):
        """filler lines until the next line starts at `target` (or one byte later, off a seam)"""
        while target - len(self.buf) > 90:
            self.filler_line()
        k = target - len(self.buf)
        if k > 0:
            body = bytes(self.rng.choice(b"abcXYZ019_ ") for _ in range(k - 1))
            self.line(body)

    def data(self):
        return bytes(self.buf)


def set_history_corpus(D, seed=0, n_big=24):
    """Family A: lines with exactly D distinct [^\\w]+ tokens, each written twice (the second pass shuffled and with
    other letter cases that lower() folds together), 300-1900 bytes long, half of them starting in the last 100
    bytes before a strip or tile seam. Returns (data, [(offset, length) of the D lines])."""
    rng = random.Random(seed * 1000 + D)
    w = Writer(rng)
    big = []
    letters = "abcdefghijklmnopqrstuvwxyz"
    if D <= 65:
        pool = set()
        while len(pool) < D:
            pool.add("".join(rng.choice(letters + "0123456789_") for _ in range(rng.randint(3, 8))))
    else:
        sym = letters + "0123456789_"
        pool = set(sym) | set(a + b for a in sym for b in sym)
    pool = sorted(pool)
    seps = [" ", ", ", ".", "-", " (", ") ", "  ", "/"]

    def case(t):
        return "".join(c.upper() if rng.random() < 0.5 else c for c in t)
    for i in range(n_big):
        for _ in range(rng.randint(1, 6)):
            w.filler_line()
        if i % 2 == 0:
            seam = V_OWN if i % 4 == 0 else V_STRIP
            nxt = (len(w.buf) // seam + 1) * seam
            w.pad_to(nxt - rng.randint(2, 99))
        words = rng.sample(pool, D)
        again = list(words)
        rng.shuffle(again)
        toks = [case(t) for t in words] + [case(t) for t in again]
        body = "".join(t + rng.choice(seps) for t in toks).encode("ascii")
        if len(body) < 300:
            body += b" " * (300 - len(body))
        off = len(w.buf)
        w.line(body)
        big.append((off, len(w.buf) - off - 1))
    for _ in range(20):
        w.filler_line()
    return w.data(), big


D_VALUES = (31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257)


def token_seam_corpus(seed=1, n_tiles=26):
    """Family B: tokens planted on the strip seams. Every tile seam and every seam 2 KB past one (the end of the
    previous tile's window in a whole-range call) is crossed by a token of 8-13 bytes at each of the four
    alignments; the other seams are crossed by, or end, tokens of 1-16, 40 and 200 bytes. Separators are every
    str.split whitespace byte but '\\r'; some short tokens hold a NUL or 0x7F; tokens of 5000 bytes sit early in a
    tile. Returns (data, [(seam, token start, token length)])."""
    rng = random.Random(seed)
    seps = [b" ", b"\t", b"\x0b", b"\x0c", b"\x1c", b"\x1d", b"\x1e", b"\x1f"]
    buf = bytearray()
    planted = []
    combos = [(L, a) for L in range(8, 14) for a in range(4)]
    others = [(L, a, rel) for L in list(range(1, 17)) + [40, 200] for a in range(4) for rel in ("cross", "end")]
    rng.shuffle(others)
    oi = 0

    def word(L):
        t = bytes(rng.choice(WORD) for _ in range(L))
        if L >= 2 and rng.random() < 0.1:
            t = t[:L - 1] + rng.choice([b"\0", b"\x7f"]) if rng.random() < 0.5 else rng.choice([b"\0", b"\x7f"]) + t[1:]
        return t

    def fill_to(pos):
        """filler words and newlines up to pos; byte pos - 1 is a separator"""
        since_nl = 0
        while len(buf) < pos:
            room = pos - len(buf)
            if room <= 2:
                buf.extend(b" " * room)
                break
            L = min(rng.randint(1, 12), room - 1)
            buf.extend(word(L))
            since_nl += L + 1
            if since_nl > rng.randint(30, 300) or rng.random() < 0.01:
                buf.extend(b"\n")
                since_nl = 0
            else:
                buf.extend(rng.choice(seps))
        assert len(buf) == pos
        if buf[pos - 1:pos] not in seps and buf[pos - 1:pos] != b"\n":
            buf[pos - 1:pos] = b" "

    for j in range(1, 8 * n_tiles):
        s = j * V_STRIP
        if j % 8 == 0:
            L, a = combos[(j // 8 - 1) % len(combos)]
            rel = "cross"
        elif j % 8 == 1:
            L, a = combos[(j // 8) % len(combos)]
            rel = "cross"
        else:
            L, a, rel = others[oi % len(others)]
            oi += 1
        if rel == "end":
            start = s - L
        else:
            ks = [k for k in range(1, L) if (s - k) % 4 == a] or [k for k in range(1, L)] or [0]
            start = s - rng.choice(ks)
        if j % 8 == 2 and j // 8 % 3 == 0:
            # a 5000-byte token early in the tile (its line fits the window of the tile it starts in)
            fill_to(len(buf) + 8)
            buf.extend(b"Q" * 5000 + b"\n")
            continue
        if start <= len(buf) + 1:
            continue
        fill_to(start)
        tok = word(L)
        buf.extend(tok)
        planted.append((s, start, L))
        buf.extend(rng.choice(seps))
    # NUL and DEL inside short str.split tokens next to the same token without them, and "a\0" next to "a"
    buf.extend(b"\na\0 a a\0 \0a a\x7f ab\0cd abcd a\0b\0c\0d\0e A\n")
    return bytes(buf), planted


def long_token_corpus(seed=2, n_tokens=100000, n_vocab=5000):
    """Family C: about 5,000 distinct str.split tokens of 10-40 bytes that share 9-30-byte prefixes, with pairs that
    differ only in their last byte or by one extra trailing byte, Zipf-repeated. Returns (data, vocabulary)."""
    rng = random.Random(seed)
    alnum = b"abcdefghijklmnopqrstuvwxyz0123456789"
    vocab = set()
    while len(vocab) < n_vocab:
        p = bytes(rng.choice(alnum) for _ in range(rng.randint(9, 30)))
        for _ in range(rng.randint(2, 12)):
            t = p + bytes(rng.choice(alnum) for _ in range(rng.randint(1, max(1, 40 - len(p)))))
            t = t[:40]
            vocab.add(t)
            vocab.add(t[:-1] + bytes([t[-1] ^ 1]) if t[-1] ^ 1 in alnum else t[:-1] + b"z")
            if len(t) < 40:
                vocab.add(t + b"x")
    vocab = sorted(v for v in vocab if 10 <= len(v) <= 40)
    rng.shuffle(vocab)
    weights = [1.0 / (i + 1) for i in range(len(vocab))]
    toks = rng.choices(vocab, weights=weights, k=n_tokens)
    toks[:len(vocab)] = vocab                    # every token at least once
    rng.shuffle(toks)
    lines, i = [], 0
    while i < len(toks):
        k = rng.randint(1, 15)
        lines.append(b" ".join(toks[i:i + k]) + rng.choice([b"", b" ", b" short tok"]))
        i += k
    return b"\n".join(lines) + b"\n", vocab


def bad_line_corpus(seed=3, n_strips=40, max_bad=8):
    """Family D: ASCII lines of 20-180 bytes; in a whole-range call strip k holds k % (max_bad + 1) lines the
    [^\\w]+ tokenisers hand to the host (non-ASCII or '\\r'), the bad byte first, last or inside, some of them
    straddling the strip seam, CRLF and lone '\\r' lines among them, and a bad last line without '\\n'.
    Returns (data, {strip: number of bad lines starting in it in text mode})."""
    rng = random.Random(seed * 7 + max_bad)
    lines = []
    size = 0
    while size < n_strips * V_STRIP:
        body = bytes(rng.choice(WORD + b"    .,") for _ in range(rng.randint(20, 180)))
        lines.append(bytearray(body))
        size += len(body) + 1
    offs, o = [], 0
    for l in lines:
        offs.append(o)
        o += len(l) + 1
    bads = [("é".encode(), "start"), ("é".encode(), "end"), (b"\r", "end"), (b"\r", "mid"),
            ("\u00a0".encode(), "mid"), ("İ".encode(), "start"), ("ß".encode(), "end"), (b"\r", "start")]
    per = {}
    for k in range(n_strips):
        want = k % (max_bad + 1)
        idx = [i for i, x in enumerate(offs) if k * V_STRIP <= x < (k + 1) * V_STRIP]
        straddler = [i for i in idx if offs[i] + len(lines[i]) >= (k + 1) * V_STRIP]
        chosen = (straddler[:1] if k % 3 == 0 else []) + rng.sample([i for i in idx if i not in straddler], want)
        chosen = chosen[:want]
        for i in chosen:
            b, where = bads[rng.randrange(len(bads))]
            l = lines[i]
            if i in straddler and len(l) > len(b) + 1:
                p = len(l) - len(b)                      # past the seam
            elif where == "start":
                p = 0
            elif where == "end":
                p = len(l) - len(b)
            else:
                p = rng.randint(0, len(l) - len(b))
            l[p:p + len(b)] = b                          # same length: offsets stay put
        per[k] = len(chosen)
    lines[-1][-2:] = "é".encode()
    data = b"\n".join(bytes(l) for l in lines)          # the last (bad) line has no '\n'
    return data, per


def field_value_spellings():
    return ["0", "-0", "+0", "007", "+", "-", "", "5_0", " 5", "5 ", "0x10", "9" * 18, "-" + "9" * 18, "+" + "9" * 18,
            "1" + "0" * 18, "-1" + "0" * 18, "٣", "12", "-7", "+31"]


FIELD_SEPS = [ord(c) for c in ", \t|;\x0b\x7f1"]


def fields_corpus(sep, seed=4, n_lines=6000, longest=F_FB_MAXLEN):
    """Family E: lines of 1-12 fields separated by `sep`, with empty fields, str keys of 0-12 and 40 bytes and the
    int() spellings the device must refuse or take, '\\r', NUL and non-ASCII lines, and lines of 4094-4097 bytes and
    of `longest` bytes that start just before a tile seam. Returns (data, {length: offset} of the long lines)."""
    rng = random.Random(seed * 131 + sep)
    s = chr(sep)
    alnum = "abcdefghijKLMNOPQRSTuvwxyz_-."
    ints = [x for x in field_value_spellings()]
    w = Writer(rng)
    longs = {}

    def field():
        r = rng.random()
        if r < 0.45:
            return str(rng.randint(-10 ** 6, 10 ** 6))
        if r < 0.6:
            return rng.choice(ints)
        if r < 0.95:
            L = rng.choice([0, 1, 2, 3, 5, 8, 9, 10, 11, 12, 40])
            return "".join(rng.choice(alnum) for _ in range(L))
        return rng.choice(["a\rb", "x\0y", "café", "\r"])

    def one():
        f = [field() for _ in range(rng.randint(1, 12))]
        return s.join(f).encode("utf-8")
    long_lens = [4094, 4095, 4096, 4097, longest]
    step = n_lines // len(long_lens)
    for i in range(n_lines):
        if i % step == step // 2 and i // step < len(long_lens):
            L = long_lens[i // step]
            nxt = (len(w.buf) // F_OWN + 1) * F_OWN
            w.pad_to(nxt - rng.randint(8, 60))
            head = ("k%d%s12%s-34%s" % (L, s, s, s)).encode("ascii")
            body = head + b"z" * (L - len(head))
            if (len(w.buf) + len(body) + 1) % V_STRIP == 0:
                w.buf += b"a" + s.encode("ascii") + b"1\n"
            longs[L] = len(w.buf)
            w.buf += body + b"\n"
            continue
        w.line(one())
    w.buf += one()                                           # no final '\n'
    return w.data(), longs


FIELD_SPECS = [   # (key field, key kind, value field, op)
    (0, FIELD_KEY_STR, FIELD_VAL_ONE, OP_SUM_I64),
    (-1, FIELD_KEY_STR, 1, OP_SUM_I64),
    (2, FIELD_KEY_STR, -2, OP_MIN_I64),
    (1, FIELD_KEY_INT, 0, OP_MAX_I64),
    (-3, FIELD_KEY_INT, FIELD_VAL_ONE, OP_SUM_I64),
    (11, FIELD_KEY_STR, -12, OP_MAX_I64),
    (0, FIELD_KEY_INT, -1, OP_MIN_I64),
]


# ---- ownership splits ------------------------------------------------------------------------------------------------
def cut_sets(n, seed=5):
    """ownership splits of [0, n) with 16-byte-aligned cut points: the whole range, random cuts, and cuts at strip
    and tile multiples +- 16. Returns {name: [(lo, hi), ...]}."""
    rng = random.Random(seed + n)

    def ranges(points):
        pts = sorted(set(p for p in points if 0 < p < n and p % 16 == 0))
        bounds = [0] + pts + [n]
        return [(a, b) for a, b in zip(bounds, bounds[1:])]
    rand = [rng.randrange(0, n // 16 + 1) * 16 for _ in range(max(1, min(12, n // 4096)))]
    seams = []
    for m in range(V_STRIP, n, V_STRIP):
        if m % V_OWN == 0 or (m // V_STRIP) % 3 == 0:
            seams.append(m + rng.choice([-16, 16]))
    return {"whole": [(0, n)], "random": ranges(rand), "seams": ranges(seams)}
