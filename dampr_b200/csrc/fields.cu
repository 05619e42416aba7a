// fields.cu — delimited-field scan + combine: `line.split(sep)[i]` keys folded with a count, an int sum, a minimum
// or a maximum of `int(line.split(sep)[j])`, a minimum or maximum of `float(line.split(sep)[j])`, and the per-line
// records of float sums and mean().
//
// Replaces, for the lowered field idioms, the reference's per-record Python in the map stage:
//   TextLineDataset.read      dampr/dataset.py:458-476  (line ownership, '\n' stripping)
//   Map.stream(user lambdas)  dampr/base.py:30-33 with `l.split(S)[i]` keys and `1` / `int(l.split(S)[j])` values
//   ReducedWriter.add_record  dampr/dataset.py:100-105  (dict combiner with binop +, min or max)
//
// Design: persistent CTAs. A CTA copies a 16 KB tile of the text (plus a 4 KB halo) into shared memory, finds the
// lines whose first byte lies in the tile (newline masks, one block scan that compacts their starts), then gives
// one line to each thread. A thread walks its line 4 bytes per step with SWAR masks for separator, newline and the
// bytes the device does not take; it resolves the key and value fields (negative indices count the separators
// first), builds the key code, parses the value and does ONE insert into the global (L2-resident) combiner table.
// There is one table operation per line, not one per token, so no shared-memory combiner sits in front of it.
// HBM traffic = the text, read once.
//
// Key codes: a str key of 1..9 bytes packs 7 bits per byte (the str.split code of the tokeniser, so the table's
// word decoding applies unchanged); '' and longer keys take the seeded hash with bit 63 set and a representative
// (offset << 20 | length) that every later occurrence is byte-compared with (DAMPR_TF_COLLISION on a mismatch).
// '' would pack to 0, the table's empty-slot marker: it goes through the hashed path with a length-0
// representative. An int key v (|v| < 10^18) is v ^ 2^63: never 0, ordered like a signed int.
//
// Accumulators: SUM adds two's-complement values. MIN and MAX keep an order-preserving code whose identity is 0
// (the cleared table), so no entry needs initialising: MAX holds v ^ 2^63, MIN holds ~(v ^ 2^63), both folded with
// an unsigned atomicMax. `float()` values (fparse.cuh) under MIN / MAX use the order-preserving code of the double,
// bits ^ (sign ? ~0 : 2^63), the same way.
//
// Record mode (float sums, mean()): float + is not associative bit for bit, so the values are not folded here.
// The kernel writes one 16-byte record {key code, value bits} per owned line, in line order, for a sort + ordered
// segmented reduce on the caller's side; the table still takes one insert per line and counts the lines of each
// key. The record index of a line is run_base + tile_base + its index among the tile's line starts. A count pass
// (the same kernel, COUNT mode, sharing the line-start code) writes the lines per tile, one CTA scans them into
// tile bases and advances run_base (a table stats slot), then the fold pass writes the records. No CTA waits for
// another, and the records of a scan do not depend on how it is cut into ranges.
//
// WHERE (the stage's `filter(...)` calls, a compile-time parameter, so the plain scans compile as before): up to 8
// predicates travel in the kernel's parameters (WhereView, ~1.6 KB, read in place through __grid_constant__).
// Predicate j owns bound slot j; the separator walk that finds the key and value also finds every predicate's
// field, the slots unrolled at compile time so the bounds stay in registers. The predicates are then evaluated in
// chain order: the first false one drops the line before its key or value is parsed (a hole in record mode); one
// the device cannot decide sends the line to the host, whose Python filters decide or raise. A program with `and` /
// `or` / `not` (WhereProg, behind the parameters the plain builds read) evaluates every leaf to T, F or U and folds
// them left-sequentially, as Python's short circuit does (where_program); a leaf may also read the whole line.
//
// WS (`line.split()`, DAMPR_FIELD_SEP_WS, a compile-time parameter, so the single-byte scans compile as before): the
// separator mask becomes the str.split() whitespace mask (0x09-0x0D, 0x1C-0x20; '\r' only reaches it under
// cr_is_data, otherwise the line is the host's). A field starts at a non-whitespace byte whose previous byte is
// whitespace or lies before the line (the class of the last byte is carried across the 4-byte steps), and ends at
// the next whitespace byte or the line end. Pass 1 counts the starts (the field count: 0 for a blank line, so every
// index is missing), pass 2 walks the class changes: change 2i opens field i, change 2i + 1 closes it.
//
// TUP (tuple keys `(r[i], int(r[j]), ...)`, a compile-time parameter of the separator-byte and WS scans): up to 4
// components take bound slots in the same walk as the predicates. The key code streams hash_bytes' two states over
// the components (str bytes, the 8 bytes of v ^ 2^63 of an int, 0xFF between them). Components are not adjacent in
// the line, so the representative is the line itself (offset << 20 | length, atomicMin keeps the lowest); an insert
// that finds another line there splits that line again in global memory and compares the components (same_tuple).
// table_tuple_keys_kernel decodes a tuple table the same way, from each entry's representative line.
//
// JSON paths (members r["a"]["b"].., their own builds, so the top-level JSON scans compile as before): the host
// builds a trie of the wanted (parent, name) nodes. The line is validated by the same state machine, which also
// tracks the node whose object it is in and compares names only there; a node's value clears the object bits and
// member types of its subtree (the last occurrence of an interior name replaces its earlier subtree). A member whose
// nodes above are not all objects at the line's end is one Python raises on: a read of it is a host line, a
// predicate on it undecided.
#include <type_traits>

#include "common.cuh"
#include "fparse.cuh"

namespace {

constexpr int F_THREADS = 256;
constexpr int F_LEAD = 16;
constexpr int F_OWN = 16384;
constexpr int F_HALO = 4096;                      // longest line handled on the device, newline included
constexpr int F_WIN = F_LEAD + F_OWN + F_HALO;    // 20496
constexpr u32 F_G_MAX_PROBES = 1u << 14;
constexpr u32 F_FB_MAXLEN = 0xFFFFu;             // the fallback list stores 16-bit lengths

static_assert(F_WIN % 16 == 0, "window must be whole 16-byte vectors");
static_assert(F_OWN % 16 == 0 && F_LEAD % 16 == 0, "tiles must keep 16-byte alignment");
static_assert(TEXT_LEAD >= F_LEAD, "textbuf lead-in too small");
static_assert(TEXT_TAIL_PAD >= F_WIN + 64, "textbuf tail pad too small");
static_assert(TEXT_TAIL_PAD >= (int)F_FB_MAXLEN + 1, "tail pad must cover the long-line measurement");

// S_RECORDS: record mode's running record count (run_base of the next range); S_DROPPED: the same slot in table
// mode, the lines a WHERE predicate rejected
enum { S_ENTRIES = 0, S_LINES = 1, S_MAXABS = 2, S_FOLDED = 3, S_FLAGS = 4, S_LONG = 5, S_RECORDS = 6, S_FALLBACK = 7 };
enum { S_DROPPED = S_RECORDS };

enum { VK_INT = 0, VK_F64 = 1 };                      // value kind: int() or float()
enum { M_TABLE = 0, M_COUNT = 1, M_RECORDS = 2 };     // fold into the table / count lines per tile / write records
constexpr int SCAN_THREADS = 1024;

struct RecView {
    ulonglong2 *rec;
    u64 cap;
    u64 *tiles;   // M_COUNT: lines per tile (written); M_RECORDS: record index of each tile's first line (read)
};

struct FieldsView {
    u64 *keys;
    u64 *counts;
    u64 *reps;
    u64 *stats;
    u64 *fb;
    u64 mask;
    u64 seed;
    u32 fb_cap;
    u32 sep;
    int key_field;
    int val_field;   // DAMPR_FIELD_VAL_ONE: the constant 1
    int key_int;
    int op;
    u32 cr_is_data;
};

constexpr int P_MAX = DAMPR_PRED_MAX;

struct PredSlot {
    int field;           // index into the split line (negative from the end); unused for NFIELDS
    u8 kind, cmp;        // DAMPR_PRED_*, DAMPR_CMP_*
    u8 first, n;         // constants c[first, first + n)
};

// a WHERE program's entries: leaf j (< P_MAX) or a connective
enum : u8 { W_AND = 0x80, W_OR = 0x81, W_NOT = 0x82 };

// the predicates of a WHERE scan, passed by value in the kernel parameters (4 KB limit)
struct WhereView {
    PredSlot p[P_MAX];                    // the leaves; leaf j owns bound slot j
    long long c[DAMPR_PRED_MAX_CONSTS];   // INT / NFIELDS / LEN values, F64 constant bits, STR: offset << 32 | len
    u8 b[DAMPR_PRED_MAX_BYTES];           // STR constants
    int n;                                // leaves
};

// a WHERE program with connectives. It travels after the parameters a plain build reads (the tuple components, the
// expression programs), so those keep their offsets and the plain builds their code.
struct WhereProg {
    int np;                               // entries of op; 0: the leaves are an AND chain
    u8 op[P_MAX + DAMPR_PRED_MAX_OPS];    // postfix: leaf indices and W_AND / W_OR / W_NOT
};

// the parameter of the separator-byte, whitespace and JSON WHERE builds (fields_tiles finds `g` behind `v`, as it
// finds a TupleWhere's members)
struct Where {
    WhereView v;
    WhereProg g;
};
static_assert(sizeof(Where) + 256 <= 4096, "kernel parameters");

struct SmemF {
    alignas(16) u8 text[F_WIN];
    u16 starts[F_OWN];
    u32 warp_tot[F_THREADS / 32];
    u32 nstarts;
    u32 flags;
};

__device__ __forceinline__ u32 eq7(u32 x7, u32 k) {  // bit 7 of each byte set iff the (7-bit) byte == k
    u32 z = x7 ^ (k * 0x01010101u);
    return ~(z + 0x7F7F7F7Fu) & 0x80808080u;
}

__device__ __forceinline__ u32 ge7(u32 x7, u32 k) {  // bit 7 of each byte set iff the (7-bit) byte >= k
    return (x7 + (0x80u - k) * 0x01010101u) & 0x80808080u;
}

// masks (bit 7 of each byte) of the 4 bytes of w: newline, separator (WS: str.split() whitespace), byte the device
// does not take
template <bool WS>
__device__ __forceinline__ void classify(u32 w, u32 sep, bool cr_data, u32 &nl, u32 &sp, u32 &bad) {
    const u32 hi = w & 0x80808080u;
    const u32 x7 = w & 0x7F7F7F7Fu;
    nl = eq7(x7, 0x0Au) & ~hi;
    if constexpr (WS) sp = ((ge7(x7, 0x09u) & ~ge7(x7, 0x0Eu)) | (ge7(x7, 0x1Cu) & ~ge7(x7, 0x21u))) & ~hi;
    else sp = eq7(x7, sep) & ~hi;
    bad = hi | (eq7(x7, 0u) & ~hi);
    if (!cr_data) bad |= eq7(x7, 0x0Du) & ~hi;
}

// parse [+-]?[0-9]{1,18} exactly; false for anything else (Python then decides)
__device__ __forceinline__ bool parse_int(const u8 *p, u32 len, long long &out) {
    u32 i = 0;
    bool neg = false;
    if (len && (p[0] == '+' || p[0] == '-')) {
        neg = p[0] == '-';
        i = 1;
    }
    const u32 nd = len - i;
    if (nd == 0 || nd > 18) return false;
    long long v = 0;
    for (; i < len; ++i) {
        const u32 d = (u32)p[i] - '0';
        if (d > 9) return false;
        v = v * 10 + d;
    }
    out = neg ? -v : v;
    return true;
}

// c = sign of (field - constant) under an ordered comparison EQ .. GE
__device__ __forceinline__ bool cmp_holds(int cmp, int c) {
    switch (cmp) {
        case DAMPR_CMP_EQ: return c == 0;
        case DAMPR_CMP_NE: return c != 0;
        case DAMPR_CMP_LT: return c < 0;
        case DAMPR_CMP_LE: return c <= 0;
        case DAMPR_CMP_GT: return c > 0;
        default: return c >= 0;
    }
}

// byte order of the field p[0, len) against STR constant k (UTF-8 byte order is code-point order, as Python's)
__device__ __forceinline__ int str_order(const WhereView &w, const u8 *p, u32 len, long long k) {
    const u8 *s = w.b + (k >> 32);
    const u32 kl = (u32)k;
    const u32 m = min(len, kl);
    for (u32 i = 0; i < m; ++i)
        if (p[i] != s[i]) return p[i] < s[i] ? -1 : 1;
    return len < kl ? -1 : (len > kl ? 1 : 0);
}

// `s in p[0, len)` for a constant s of kl bytes: a scan of aligned words of the field in shared memory for s's first
// byte, then a byte compare at each hit. O(len * kl) at worst (4 KB x 1 KB).
__device__ __forceinline__ bool contains(const u8 *p, u32 len, const u8 *s, u32 kl) {
    if (kl == 0) return true;
    if (kl > len) return false;
    const u32 a = (u32)(uintptr_t)p & 3u, hi = a + len - kl + 1;   // candidate starts: word bytes [a, hi)
    const u8 *base = p - a;
    const u32 k0 = s[0] * 0x01010101u;
    for (u32 o = 0; o < hi; o += 4) {
        u32 m = __vcmpeq4(*reinterpret_cast<const u32 *>(base + o), k0);
        if (o == 0) m &= ~0u << (8 * a);
        if (o + 4 > hi) m &= (1u << (8 * (hi - o))) - 1u;
        while (m) {
            const u32 b = ((u32)__ffs(m) - 1u) >> 3, i = o + b - a;
            m &= ~(0xFFu << (8 * b));   // __vcmpeq4 sets all 8 bits of a hit
            u32 j = 1;
            while (j < kl && p[i + j] == s[j]) ++j;
            if (j == kl) return true;
        }
    }
    return false;
}

// p[0, len) holds a byte outside the str.split() whitespace class (`x.strip()` is truthy)
__device__ __forceinline__ bool nonblank(const u8 *p, u32 len) {
    const u32 a = (u32)(uintptr_t)p & 3u, hi = a + len;
    const u8 *base = p - a;
    for (u32 o = 0; o < hi; o += 4) {
        u32 nl, ws, bd;
        classify<true>(*reinterpret_cast<const u32 *>(base + o), 0u, true, nl, ws, bd);
        u32 keep = 0x80808080u;
        if (o == 0) keep &= ~0u << (8 * a);
        if (o + 4 > hi) keep &= (1u << (8 * (hi - o))) - 1u;
        if (~ws & keep) return true;
    }
    return false;
}

// one predicate over its field p[0, len) (nf: the line's field count): 1 true, 0 false, -1 for the host to decide
// (no such field, or an int() / float() field the device does not parse exactly)
__device__ __noinline__ int eval_pred(const WhereView &w, const PredSlot &pr, bool has, const u8 *p, u32 len,
                                      int nf) {
    if (pr.kind == DAMPR_PRED_NFIELDS) return cmp_holds(pr.cmp, nf < w.c[pr.first] ? -1 : nf > w.c[pr.first]);
    if (!has) return -1;   // IndexError in Python
    if (pr.kind == DAMPR_PRED_LEN) return cmp_holds(pr.cmp, len < w.c[pr.first] ? -1 : len > w.c[pr.first]);
    if (pr.kind == DAMPR_PRED_NONBLANK) return nonblank(p, len);
    if (pr.cmp >= DAMPR_CMP_CONTAINS) {   // STR: substring, prefix, suffix
        if (pr.cmp <= DAMPR_CMP_NOT_CONTAINS) {
            const long long k = w.c[pr.first];
            return contains(p, len, w.b + (k >> 32), (u32)k) == (pr.cmp == DAMPR_CMP_CONTAINS);
        }
        for (int i = pr.first; i < pr.first + pr.n; ++i) {
            const u8 *s = w.b + (w.c[i] >> 32);
            const u32 kl = (u32)w.c[i];
            if (kl > len) continue;
            const u8 *q = pr.cmp == DAMPR_CMP_STARTS ? p : p + len - kl;
            u32 j = 0;
            while (j < kl && q[j] == s[j]) ++j;
            if (j == kl) return 1;
        }
        return 0;
    }
    const bool in = pr.cmp == DAMPR_CMP_IN || pr.cmp == DAMPR_CMP_NOT_IN;
    bool r = false;
    if (pr.kind == DAMPR_PRED_F64) {
        double x;
        if (!parse_f64(p, len, x)) return -1;
        const double k = __longlong_as_double(w.c[pr.first]);
        switch (pr.cmp) {   // IEEE comparisons: NaN is false under all but !=, -0.0 == 0.0, as in Python
            case DAMPR_CMP_EQ: return x == k;
            case DAMPR_CMP_NE: return x != k;
            case DAMPR_CMP_LT: return x < k;
            case DAMPR_CMP_LE: return x <= k;
            case DAMPR_CMP_GT: return x > k;
            default: return x >= k;
        }
    }
    if (pr.kind == DAMPR_PRED_INT) {
        long long x;
        if (!parse_int(p, len, x)) return -1;
        if (!in) return cmp_holds(pr.cmp, x < w.c[pr.first] ? -1 : x > w.c[pr.first]);
        for (int i = pr.first; i < pr.first + pr.n && !r; ++i) r = x == w.c[i];
    } else {
        if (!in) return cmp_holds(pr.cmp, str_order(w, p, len, w.c[pr.first]));
        for (int i = pr.first; i < pr.first + pr.n && !r; ++i)
            r = (u32)w.c[i] == len && str_order(w, p, len, w.c[i]) == 0;
    }
    return r == (pr.cmp == DAMPR_CMP_IN);
}

// the verdict of a WHERE program (1 T, 0 F, -1 U) from its leaves' results: bit j of t / u says leaf j is T / U.
// A stack of three-valued bits (top at bit 0) under left-sequential logic, Python's short circuit: `a and b` is a
// when a is F or U, else b; `a or b` is a when a is T or U, else b; `not` keeps U. The values left are ANDed bottom
// first (one per filter call).
__device__ __forceinline__ int where_program(const WhereProg &g, u32 t, u32 u) {
    u32 st = 0, su = 0;
    int d = 0;
    for (int k = 0; k < g.np; ++k) {
        const u32 op = g.op[k];
        if (op < (u32)P_MAX) {
            st = (st << 1) | ((t >> op) & 1u);
            su = (su << 1) | ((u >> op) & 1u);
            ++d;
        } else if (op == W_NOT) {
            st ^= ~su & 1u;
        } else {
            const u32 bt = st & 1u, bu = su & 1u;
            st >>= 1;
            su >>= 1;
            --d;
            if (!(su & 1u) && (st & 1u) == (op == W_AND ? 1u : 0u)) {   // a does not decide: the result is b
                st = (st & ~1u) | bt;
                su = (su & ~1u) | bu;
            }
        }
    }
    const u32 open = ~st & ((1u << d) - 1u);   // the values that are not T
    if (!open) return 1;
    return (su >> (31 - __clz(open))) & 1u ? -1 : 0;
}

// ---- JSON lines ------------------------------------------------------------------------------------------------
constexpr int J_MAX = DAMPR_JSON_MAX_MEMBERS;
constexpr int J_NAME = DAMPR_JSON_MAX_NAME;
constexpr int J_DEPTH = DAMPR_JSON_MAX_DEPTH;
static_assert(J_DEPTH <= 64, "the container stack is one u64");
static_assert(F_WIN <= 0xFFFF, "member bounds pack two 16-bit window positions");

// the JSON type of a member, 4 bits per member in one u32 (NONE: not in the line)
enum { JT_NONE = 0, JT_STR = 1, JT_ESC = 2, JT_INT = 3, JT_FLOAT = 4, JT_OTHER = 5 };

// the wanted member names of a JSON scan, passed by value in the kernel parameters
struct JsonView {
    u8 name[J_MAX][J_NAME];
    u8 len[J_MAX];
    int n;
};

// first position >= i whose byte is not an ASCII digit (the line's '\n' stops it)
__device__ __forceinline__ u32 skip_digits(const u8 *t, u32 i) {
    for (;;) {
        const u32 a = i & ~3u;
        const u32 x7 = *reinterpret_cast<const u32 *>(t + a) & 0x7F7F7F7Fu;
        const u32 nd = ~(ge7(x7, '0') & ~ge7(x7, '9' + 1)) & 0x80808080u & (~0u << (8 * (i - a)));
        if (nd) return a + (((u32)__ffs(nd) - 1u) >> 3);
        i = a + 4;
    }
}

// first position >= i whose byte is '"', '\\' or below 0x20 (the line's '\n' stops it)
__device__ __forceinline__ u32 skip_string(const u8 *t, u32 i) {
    for (;;) {
        const u32 a = i & ~3u;
        const u32 x7 = *reinterpret_cast<const u32 *>(t + a) & 0x7F7F7F7Fu;
        const u32 sp = (eq7(x7, '"') | eq7(x7, '\\') | ~ge7(x7, 0x20u)) & 0x80808080u & (~0u << (8 * (i - a)));
        if (sp) return a + (((u32)__ffs(sp) - 1u) >> 3);
        i = a + 4;
    }
}

__device__ __forceinline__ bool is_digit(u8 c) { return (u32)c - '0' <= 9u; }
__device__ __forceinline__ bool is_hex(u8 c) { return is_digit(c) || (u32)(c | 0x20) - 'a' <= 5u; }

// t[p, end) against the bytes of lit (json.loads' true / false / null)
__device__ __forceinline__ bool lit_at(const u8 *t, u32 p, u32 end, const char *lit, u32 n) {
    if (p + n > end) return false;
    for (u32 i = 0; i < n; ++i)
        if (t[p + i] != (u8)lit[i]) return false;
    return true;
}

// the JSON string whose opening quote is at p: *e = the position of its closing quote, *esc = it holds an escape;
// false when json.loads rejects it (a bad escape, a raw byte below 0x20, no closing quote before the line end)
__device__ __forceinline__ bool json_string(const u8 *t, u32 p, u32 end, u32 &e, bool &esc) {
    esc = false;
    for (e = p + 1;;) {
        e = skip_string(t, e);
        if (e >= end || t[e] < 0x20) return false;
        if (t[e] == '"') return true;
        esc = true;
        const u8 x = t[e + 1];
        if (x == 'u') {
            if (e + 6 > end || !is_hex(t[e + 2]) || !is_hex(t[e + 3]) || !is_hex(t[e + 4]) || !is_hex(t[e + 5]))
                return false;
            e += 6;
        } else if (x == '"' || x == '\\' || x == '/' || x == 'b' || x == 'f' || x == 'n' || x == 'r' || x == 't') {
            e += 2;
        } else {
            return false;
        }
    }
}

// Validate the line t[q, end) (t[end] == '\n'; every byte ASCII, not NUL, '\r' only where it is data) as one JSON
// text whose top-level value is an object, under json.loads' grammar, and record the last occurrence of each wanted
// top-level member: mb[j] = start | end << 16 of its value (a string's bytes between the quotes), its JT_* type in
// bits 4j of mt. false for anything json.loads rejects (the host raises), a nesting deeper than J_DEPTH, and a
// top-level name with an escape (it might decode to a wanted name).
template <int JM>
__device__ __forceinline__ bool json_line(const u8 *t, u32 q, u32 end, const JsonView &jv, u32 (&mb)[JM], u32 &mt) {
    enum { VALUE, VALUE_OR_CLOSE, NAME, NAME_OR_CLOSE, COLON, AFTER };
    u64 objs = 0;     // bit d - 1: the container at depth d is an object
    int depth = 0;
    int st = VALUE;
    int cur = -1;     // the wanted member whose value comes next (depth 1)
    u32 p = q;
    while (p < end) {
        const u8 c = t[p];
        if (c == ' ' || c == '\t' || c == '\r') {   // '\r' is only here when it is data: JSON whitespace
            ++p;
            continue;
        }
        if (st == NAME_OR_CLOSE && c == '}') {
            objs &= ~(1ULL << --depth);
            st = AFTER;
            ++p;
            continue;
        }
        if (st == NAME_OR_CLOSE || st == NAME) {
            u32 e;
            bool esc;
            if (c != '"' || !json_string(t, p, end, e, esc)) return false;
            if (depth == 1) {
                if (esc) return false;
                const u32 len = e - p - 1;
                cur = -1;
#pragma unroll
                for (int j = 0; j < JM; ++j) {
                    if (j < jv.n && cur < 0 && len == jv.len[j]) {
                        bool same = true;
                        for (u32 i = 0; i < len && same; ++i) same = t[p + 1 + i] == jv.name[j][i];
                        if (same) cur = j;
                    }
                }
            }
            p = e + 1;
            st = COLON;
            continue;
        }
        if (st == COLON) {
            if (c != ':') return false;
            ++p;
            st = VALUE;
            continue;
        }
        if (st == AFTER) {
            if (depth == 0) return false;   // data after the top-level object
            const bool obj = (objs >> (depth - 1)) & 1;
            if (c == ',') st = obj ? NAME : VALUE;
            else if (c == (obj ? '}' : ']')) objs &= ~(1ULL << --depth);
            else return false;
            ++p;
            continue;
        }
        // a value (VALUE, VALUE_OR_CLOSE)
        if (st == VALUE_OR_CLOSE && c == ']') {
            --depth;
            st = AFTER;
            ++p;
            continue;
        }
        if (depth == 0 && c != '{') return false;   // the top-level value is an object
        const bool member = depth == 1 && cur >= 0;
        u32 vs = p;
        int ty = JT_OTHER;
        st = AFTER;
        if (c == '{' || c == '[') {
            if (depth == J_DEPTH) return false;
            if (c == '{') objs |= 1ULL << depth;
            ++depth;
            st = c == '{' ? NAME_OR_CLOSE : VALUE_OR_CLOSE;
            ++p;
        } else if (c == '"') {
            u32 e;
            bool esc;
            if (!json_string(t, p, end, e, esc)) return false;
            ty = esc ? JT_ESC : JT_STR;
            vs = p + 1;
            p = e;   // the bounds end at the closing quote, the scan goes on after it
        } else if (c == '-' || is_digit(c)) {
            u32 i = p + (c == '-');
            if (t[i] == '0') ++i;
            else if (is_digit(t[i])) i = skip_digits(t, i + 1);
            else return false;
            ty = JT_INT;
            if (t[i] == '.') {
                if (!is_digit(t[i + 1])) return false;
                i = skip_digits(t, i + 2);
                ty = JT_FLOAT;
            }
            if ((t[i] | 0x20) == 'e') {
                ++i;
                if (t[i] == '+' || t[i] == '-') ++i;
                if (!is_digit(t[i])) return false;
                i = skip_digits(t, i + 1);
                ty = JT_FLOAT;
            }
            p = i;
        } else {
            const u32 n = c == 'f' ? 5u : 4u;
            if (!lit_at(t, p, end, c == 't' ? "true" : c == 'f' ? "false" : "null", n)) return false;
            p += n;
        }
        if (member) {
#pragma unroll
            for (int j = 0; j < JM; ++j)
                if (j == cur) {
                    mb[j] = vs | p << 16;
                    mt = (mt & ~(0xFu << (4 * j))) | (u32)ty << (4 * j);
                }
        }
        if (ty == JT_STR || ty == JT_ESC) ++p;   // past the closing quote
    }
    return st == AFTER && depth == 0;
}

// member j's entry of the packed bounds (unrolled: mb stays in registers)
template <int JM>
__device__ __forceinline__ u32 member_bounds(const u32 (&mb)[JM], int j) {
    u32 b = 0;
#pragma unroll
    for (int i = 0; i < JM; ++i)
        if (i == j) b = mb[i];
    return b;
}

// ---- JSON paths: members r[n1]..[nk] ---------------------------------------------------------------------------
constexpr int J_NODES = DAMPR_JSON_MAX_NODES;
static_assert(J_NODES <= 16 && J_MAX <= 8, "node masks are u16, member type nibbles one u32");

// the wanted paths of a JSON scan as a trie of (parent, name) nodes, passed by value in the kernel parameters
struct JsonPathView {
    u8 name[J_NODES][J_NAME];
    u8 len[J_NODES];
    signed char up[J_NODES];     // the parent node, -1 for a top-level name
    signed char leaf[J_NODES];   // the member this node's value is, or -1
    u16 kids[J_NODES + 1];       // kids[k + 1]: the nodes whose parent is k; kids[0]: the top-level names
    u16 sub[J_NODES];            // the nodes beneath k
    u32 sub_types[J_NODES];      // the type nibbles (of mt) of the members beneath k
    u16 anc[J_MAX];              // the nodes above member j's own
    signed char up_leaf[J_MAX];  // the member that is member j's parent node, or -1
    int n;                       // members
};

// json_line over paths: the same validation, with names compared in the top-level object and in the object of each
// interior node on a wanted path (an escaped name there returns false). A node's value replaces its earlier
// occurrence's whole subtree. On return, member j's type is JT_NONE and bit j of bad is set when a node above it is
// not an object in the line (missing, or its last occurrence is not an object): Python raises on reading it.
template <int JM>
__device__ __forceinline__ bool json_path_line(const u8 *t, u32 q, u32 end, const JsonPathView &jv, u32 (&mb)[JM],
                                               u32 &mt, u32 &bad) {
    enum { VALUE, VALUE_OR_CLOSE, NAME, NAME_OR_CLOSE, COLON, AFTER };
    u64 objs = 0;     // bit d - 1: the container at depth d is an object
    int depth = 0;
    int st = VALUE;
    int node = -1;    // the node whose object the scan compares names in (-1: the top-level object)
    int nd = 1;       // that object's depth
    int cur = -1;     // the child of node whose value comes next (depth nd)
    u32 obj = 0;      // bit k: node k's last occurrence so far is an object
    u32 p = q;
    while (p < end) {
        const u8 c = t[p];
        if (c == ' ' || c == '\t' || c == '\r') {
            ++p;
            continue;
        }
        if ((st == NAME_OR_CLOSE || st == AFTER) && c == '}' && depth == nd && node >= 0) {
            node = jv.up[node];   // leaving a wanted node's object (its '}' is checked below)
            --nd;
            cur = -1;
        }
        if (st == NAME_OR_CLOSE && c == '}') {
            objs &= ~(1ULL << --depth);
            st = AFTER;
            ++p;
            continue;
        }
        if (st == NAME_OR_CLOSE || st == NAME) {
            u32 e;
            bool esc;
            if (c != '"' || !json_string(t, p, end, e, esc)) return false;
            if (depth == nd) {
                if (esc) return false;
                const u32 len = e - p - 1;
                cur = -1;
                for (u32 km = jv.kids[node + 1]; km && cur < 0; km &= km - 1) {
                    const int k = __ffs(km) - 1;
                    if (len != jv.len[k]) continue;
                    bool same = true;
                    for (u32 i = 0; i < len && same; ++i) same = t[p + 1 + i] == jv.name[k][i];
                    if (same) cur = k;
                }
            }
            p = e + 1;
            st = COLON;
            continue;
        }
        if (st == COLON) {
            if (c != ':') return false;
            ++p;
            st = VALUE;
            continue;
        }
        if (st == AFTER) {
            if (depth == 0) return false;
            const bool ob = (objs >> (depth - 1)) & 1;
            if (c == ',') st = ob ? NAME : VALUE;
            else if (c == (ob ? '}' : ']')) objs &= ~(1ULL << --depth);
            else return false;
            ++p;
            continue;
        }
        if (st == VALUE_OR_CLOSE && c == ']') {
            --depth;
            st = AFTER;
            ++p;
            continue;
        }
        if (depth == 0 && c != '{') return false;
        const int k = depth == nd ? cur : -1;   // the wanted node this value belongs to
        if (k >= 0) {   // a new occurrence: forget the earlier one's subtree
            obj = (obj & ~(u32)jv.sub[k] & ~(1u << k)) | (u32)(c == '{') << k;
            mt &= ~jv.sub_types[k];
        }
        u32 vs = p;
        int ty = JT_OTHER;
        st = AFTER;
        if (c == '{' || c == '[') {
            if (depth == J_DEPTH) return false;
            if (c == '{') objs |= 1ULL << depth;
            ++depth;
            st = c == '{' ? NAME_OR_CLOSE : VALUE_OR_CLOSE;
            ++p;
            if (k >= 0 && c == '{' && jv.kids[k + 1]) {   // descend into a wanted interior node
                node = k;
                nd = depth;
                cur = -1;
            }
        } else if (c == '"') {
            u32 e;
            bool esc;
            if (!json_string(t, p, end, e, esc)) return false;
            ty = esc ? JT_ESC : JT_STR;
            vs = p + 1;
            p = e;
        } else if (c == '-' || is_digit(c)) {
            u32 i = p + (c == '-');
            if (t[i] == '0') ++i;
            else if (is_digit(t[i])) i = skip_digits(t, i + 1);
            else return false;
            ty = JT_INT;
            if (t[i] == '.') {
                if (!is_digit(t[i + 1])) return false;
                i = skip_digits(t, i + 2);
                ty = JT_FLOAT;
            }
            if ((t[i] | 0x20) == 'e') {
                ++i;
                if (t[i] == '+' || t[i] == '-') ++i;
                if (!is_digit(t[i])) return false;
                i = skip_digits(t, i + 1);
                ty = JT_FLOAT;
            }
            p = i;
        } else {
            const u32 n = c == 'f' ? 5u : 4u;
            if (!lit_at(t, p, end, c == 't' ? "true" : c == 'f' ? "false" : "null", n)) return false;
            p += n;
        }
        if (k >= 0) {
            const int lf = jv.leaf[k];
#pragma unroll
            for (int j = 0; j < JM; ++j)
                if (j == lf) {
                    mb[j] = vs | p << 16;
                    mt = (mt & ~(0xFu << (4 * j))) | (u32)ty << (4 * j);
                }
        }
        if (ty == JT_STR || ty == JT_ESC) ++p;
    }
    if (st != AFTER || depth != 0) return false;
#pragma unroll
    for (int j = 0; j < JM; ++j)
        if (j < jv.n && (jv.anc[j] & ~obj)) {
            bad |= 1u << j;
            mt &= ~(0xFu << (4 * j));
        }
    return true;
}

__device__ __forceinline__ u64 hash_bytes(const u8 *p, u32 len, u64 seed) {
    u32 h1 = (u32)seed ^ 0x811C9DC5u, h2 = (u32)(seed >> 32) ^ 0x9747B28Cu;
    for (u32 i = 0; i < len; ++i) {
        const u32 v = p[i];
        h1 = (h1 ^ v) * 16777619u;
        h2 = (h2 ^ v) * 0x85EBCA6Bu + 0x9E3779B9u;
        h2 = (h2 << 13) | (h2 >> 19);
    }
    return mix64((((u64)h1) << 32 | h2) ^ ((u64)len * 0x9E3779B97F4A7C15ULL)) | 0x8000000000000000ULL;
}

// ---- tuple keys ------------------------------------------------------------------------------------------------
constexpr int T_MAX = DAMPR_FIELD_KEYS_MAX;

// the components of a tuple-key scan, passed by value in the kernel parameters
struct TupleView {
    int field[T_MAX];
    int is_int[T_MAX];
    int n;
};

// the parameters of a tuple-key build: its predicates (n = 0 in a plain build), components and WHERE program.
// fields_tiles takes the address of `where` (a pointer to the first member of this standard-layout struct) and finds
// `tup` and `prog` behind it.
struct TupleWhere {
    WhereView where;
    TupleView tup;
    WhereProg prog;
};

// ---- computed keys and values ----------------------------------------------------------------------------------
constexpr int X_OPS = DAMPR_EXPR_MAX_OPS;
constexpr int X_DEPTH = DAMPR_EXPR_MAX_DEPTH;
constexpr int X_CONSTS = DAMPR_EXPR_MAX_CONSTS;
constexpr long long X_I64_MIN = (long long)0x8000000000000000ULL, X_I64_MAX = 0x7FFFFFFFFFFFFFFFLL;
static_assert(DAMPR_EXPR_MAX_LOADS == T_MAX, "load slots take the tuple components' bound slots");

// the programs of an expression scan (checked on the host: every operand is there and of its type), passed by value
// in the kernel parameters; the load slots' fields are the TupleView's
struct ExprView {
    int key_len, val_len;   // 0: the spec's key / value
    int key_prog[X_OPS], val_prog[X_OPS];
    long long ci[X_CONSTS];
    double cf[X_CONSTS];
    int load_kind[T_MAX];
};

// the parameters of an expression build: fields_tiles finds `tup` (the load slots) where a tuple build does, and `ex`
// and `prog` behind it
struct ExprWhere {
    WhereView where;
    TupleView tup;
    ExprView ex;
    WhereProg prog;
};

// the value of load slot j (unrolled: the slots stay in registers)
__device__ __forceinline__ long long load_slot(const long long (&lv)[T_MAX], int j) {
    long long v = 0;
#pragma unroll
    for (int i = 0; i < T_MAX; ++i)
        if (i == j) v = lv[i];
    return v;
}

__device__ __forceinline__ double as_f(long long x) { return __longlong_as_double(x); }
__device__ __forceinline__ long long as_i(double x) { return __double_as_longlong(x); }

// run one program over the line's loads lv and field count nf: false where CPython raises or leaves int64 (the line
// is the host's); out holds an int64 or the bits of a double. Every float operation is one IEEE rounding (the
// intrinsics keep ptxas from contracting a * b + c).
__device__ __noinline__ bool eval_expr(const ExprView &ex, const int *prog, int len, long long l0, long long l1,
                                       long long l2, long long l3, int nf, long long &out) {
    const long long lv[T_MAX] = {l0, l1, l2, l3};
    constexpr long long LIM53 = 1LL << 53;
    long long st[X_DEPTH];
    int sp = 0;
    for (int pc = 0; pc < len; ++pc) {
        const int w = prog[pc], op = w & 0xFF, arg = w >> 8;
        if (op == EV_CI || op == EV_CF || op == EV_LOAD || op == EV_NF) {
            st[sp++] = op == EV_CI ? ex.ci[arg] : op == EV_CF ? as_i(ex.cf[arg]) : op == EV_LOAD ? load_slot(lv, arg)
                                                                                                : (long long)nf;
            continue;
        }
        long long &b = st[sp - 1];
        switch (op) {   // unary operations
            case EV_I2F: b = as_i(__ll2double_rn(b)); continue;
            case EV_INEG:
                if (b == X_I64_MIN) return false;
                b = -b;
                continue;
            case EV_IABS:
                if (b == X_I64_MIN) return false;
                b = b < 0 ? -b : b;
                continue;
            case EV_FNEG: b ^= X_I64_MIN; continue;
            case EV_FABS: b &= X_I64_MAX; continue;
            case EV_F2I: {   // int(x): a NaN or an infinity raises, a float outside int64 is a big int
                const double x = as_f(b);
                if (!(x >= -9223372036854775808.0 && x < 9223372036854775808.0)) return false;
                b = __double2ll_rz(x);
                continue;
            }
            default: break;
        }
        long long &a = st[sp - 2];
        --sp;
        switch (op) {
            case EV_IADD: {
                const long long r = (long long)((u64)a + (u64)b);
                if (((a ^ r) & (b ^ r)) < 0) return false;
                a = r;
                break;
            }
            case EV_ISUB: {
                const long long r = (long long)((u64)a - (u64)b);
                if (((a ^ b) & (a ^ r)) < 0) return false;
                a = r;
                break;
            }
            case EV_IMUL: {
                const long long lo = (long long)((u64)a * (u64)b);
                if (__mul64hi(a, b) != (lo >> 63)) return false;
                a = lo;
                break;
            }
            case EV_IDIV:   // int / int: CPython divides the doubles when both operands are within 2^53
                if (b == 0 || a > LIM53 || a < -LIM53 || b > LIM53 || b < -LIM53) return false;
                a = as_i(__ddiv_rn(__ll2double_rn(a), __ll2double_rn(b)));
                break;
            case EV_IFLOOR: {
                if (b == 0 || (a == X_I64_MIN && b == -1)) return false;
                long long q = a / b;
                if (q * b != a && ((a < 0) != (b < 0))) --q;
                a = q;
                break;
            }
            case EV_IMOD: {
                if (b == 0) return false;
                long long r = b == -1 ? 0 : a % b;
                if (r != 0 && ((r < 0) != (b < 0))) r += b;
                a = r;
                break;
            }
            case EV_FADD: a = as_i(__dadd_rn(as_f(a), as_f(b))); break;
            case EV_FSUB: a = as_i(__dsub_rn(as_f(a), as_f(b))); break;
            case EV_FMUL: a = as_i(__dmul_rn(as_f(a), as_f(b))); break;
            default:   // EV_FDIV
                if (as_f(b) == 0.0) return false;
                a = as_i(__ddiv_rn(as_f(a), as_f(b)));
                break;
        }
    }
    out = st[0];
    return true;
}

// a CTA's hot-key slots of an expression scan with a key program: key codes and their accumulators in the table's
// encoding, folded with shared-memory atomics and inserted into the table once, after the CTA's last tile
constexpr int X_HOT = 32;
struct HotKeys {
    u64 code[X_HOT];
    u64 acc[X_HOT];
};

__device__ __forceinline__ HotKeys &hot_keys() {
    __shared__ HotKeys h;
    return h;
}

// the table's accumulator encoding of one value under op (see the header): SUM the value, MAX / MIN order codes
__device__ __forceinline__ u64 table_code(int op, long long v) {
    if (op == DAMPR_OP_SUM_I64) return (u64)v;
    const u64 ord = op == DAMPR_OP_MIN_F64 || op == DAMPR_OP_MAX_F64
                        ? (u64)v ^ (v < 0 ? ~0ULL : 0x8000000000000000ULL)
                        : (u64)v ^ 0x8000000000000000ULL;
    return op == DAMPR_OP_MAX_I64 || op == DAMPR_OP_MAX_F64 ? ord : ~ord;
}

__device__ __forceinline__ void fold_code(u64 *acc, int op, u64 c) {
    if (op == DAMPR_OP_SUM_I64) atomicAdd(acc, c);
    else atomicMax(acc, c);
}

// fold an encoded accumulator c of an int key code into the table
__device__ __forceinline__ void table_fold_code(const FieldsView &t, u64 code, u64 c, u32 &flags) {
    u64 slot = mix64(code) & t.mask;
    for (u32 probe = 0; probe < F_G_MAX_PROBES; ++probe) {
        u64 k = *((volatile u64 *)&t.keys[slot]);
        if (k == 0) {
            k = atomicCAS(&t.keys[slot], 0ULL, code);
            if (k == 0) {
                atomicAdd(&t.stats[S_ENTRIES], 1ULL);
                k = code;
            }
        }
        if (k == code) {
            fold_code(&t.counts[slot], t.op, c);
            return;
        }
        slot = (slot + 1) & t.mask;
    }
    flags |= DAMPR_TF_TABLEFULL;
}

// a tuple-key line's components: field ci[j] (-1: no component j, or it is missing: `missing`), bounds
// [cs[j], ce[j]) in the window; nothing in the other builds
template <bool TUP>
struct TupleBounds {};
template <>
struct TupleBounds<true> {
    int ci[T_MAX];
    u32 cs[T_MAX], ce[T_MAX];
    bool missing = false;
};

// hash_bytes' two running states after one more byte v
__device__ __forceinline__ void hash_step(u32 &h1, u32 &h2, u32 v) {
    h1 = (h1 ^ v) * 16777619u;
    h2 = (h2 ^ v) * 0x85EBCA6Bu + 0x9E3779B9u;
    h2 = (h2 << 13) | (h2 >> 19);
}

// the tuple's key code from its component bounds [cs[j], ce[j]) in t (see the header); false when an int()
// component is not one the device parses (the host raises or decides)
__device__ __forceinline__ bool tuple_code(const u8 *t, const u32 (&cs)[T_MAX], const u32 (&ce)[T_MAX],
                                           const TupleView &tv, u64 seed, u64 &code) {
    u32 h1 = (u32)seed ^ 0x811C9DC5u, h2 = (u32)(seed >> 32) ^ 0x9747B28Cu, len = 0;
#pragma unroll
    for (int j = 0; j < T_MAX; ++j) {
        if (j < tv.n) {
            if (j) {
                hash_step(h1, h2, 0xFFu);
                ++len;
            }
            if (tv.is_int[j]) {
                long long v;
                if (!parse_int(t + cs[j], ce[j] - cs[j], v)) return false;
                const u64 x = (u64)v ^ 0x8000000000000000ULL;
#pragma unroll
                for (int b = 0; b < 8; ++b) hash_step(h1, h2, (u32)(x >> (8 * b)) & 0xFFu);
                len += 8;
            } else {
                for (u32 i = cs[j]; i < ce[j]; ++i) hash_step(h1, h2, t[i]);
                len += ce[j] - cs[j];
            }
        }
    }
    code = mix64((((u64)h1) << 32 | h2) ^ ((u64)len * 0x9E3779B97F4A7C15ULL)) | 0x8000000000000000ULL;
    return true;
}

__device__ __forceinline__ bool is_split_ws(u32 c) { return (c - 0x09u) <= 4u || (c - 0x1Cu) <= 4u; }

// bounds [s[j], e[j]) of the tuple's components in the taken line p[0, len) (every component exists), split by
// the byte sep or (WS) by runs of str.split() whitespace, one byte at a time
template <bool WS>
__device__ __forceinline__ void line_fields(const u8 *p, u32 len, u32 sep, const TupleView &tv, u32 (&s)[T_MAX],
                                            u32 (&e)[T_MAX]) {
    int nf = WS ? 0 : 1;
    bool prev_ws = true;
    for (u32 i = 0; i < len; ++i) {
        const u32 c = p[i];
        if constexpr (WS) {
            const bool w = is_split_ws(c);
            nf += !w && prev_ws;
            prev_ws = w;
        } else {
            nf += c == sep;
        }
    }
    int want[T_MAX];
#pragma unroll
    for (int j = 0; j < T_MAX; ++j) {
        want[j] = j < tv.n ? (tv.field[j] < 0 ? tv.field[j] + nf : tv.field[j]) : -1;
        s[j] = e[j] = 0;
    }
    int f = WS ? -1 : 0;
    u32 start = 0;
    prev_ws = true;
    for (u32 i = 0; i <= len; ++i) {
        const u32 c = i < len ? p[i] : (WS ? 0x20u : sep);   // the line end closes the last field
        bool close = false;
        if constexpr (WS) {
            const bool w = is_split_ws(c);
            if (!w && prev_ws) {
                ++f;
                start = i;
            }
            close = w && !prev_ws;
            prev_ws = w;
        } else {
            close = c == sep;
        }
        if (close) {
#pragma unroll
            for (int j = 0; j < T_MAX; ++j)
                if (want[j] == f) {
                    s[j] = start;
                    e[j] = i;
                }
            if constexpr (!WS) {
                ++f;
                start = i + 1;
            }
        }
    }
}

// the guard: the components of this line (bounds in t) against those of the representative line `other` (global
// memory, taken by the device earlier, so its split cannot fail): str as bytes, int() as values
template <bool WS>
__device__ __forceinline__ bool same_tuple(const u8 *text, u64 other, const u8 *t, const u32 (&cs)[T_MAX],
                                           const u32 (&ce)[T_MAX], const TupleView &tv, u32 sep) {
    const u8 *o = text + (other >> 20);
    u32 os[T_MAX], oe[T_MAX];
    line_fields<WS>(o, (u32)(other & 0xFFFFFu), sep, tv, os, oe);
    bool same = true;
#pragma unroll
    for (int j = 0; j < T_MAX; ++j) {
        if (j < tv.n && same) {
            const u32 la = ce[j] - cs[j], lb = oe[j] - os[j];
            if (tv.is_int[j]) {
                long long a = 0, b = 0;
                same = parse_int(t + cs[j], la, a) && parse_int(o + os[j], lb, b) && a == b;
            } else {
                same = la == lb;
                for (u32 i = 0; i < la && same; ++i) same = t[cs[j] + i] == o[os[j] + i];
            }
        }
    }
    return same;
}

// fold (code -> value) into the global table; false if a hashed key's representative is a different string.
// F64: v holds the bits of a double (MIN / MAX only). LINE_REP (tuple keys): the representative is a line, and
// when the entry's is another line than rep it goes to *other for the caller's guard (same_tuple)
template <bool F64, bool LINE_REP = false>
__device__ __forceinline__ bool fold_insert(const FieldsView &t, const u8 *text, u64 code, long long v, u64 rep,
                                            u32 &flags, u64 *other = nullptr) {
    u64 slot = mix64(code) & t.mask;
    for (u32 probe = 0; probe < F_G_MAX_PROBES; ++probe) {
        u64 k = *((volatile u64 *)&t.keys[slot]);
        if (k == 0) {
            k = atomicCAS(&t.keys[slot], 0ULL, code);
            if (k == 0) {
                atomicAdd(&t.stats[S_ENTRIES], 1ULL);
                k = code;
            }
        }
        if (k == code) {
            if constexpr (F64) {
                const u64 ord = (u64)v ^ (v < 0 ? ~0ULL : 0x8000000000000000ULL);
                atomicMax(&t.counts[slot], t.op == DAMPR_OP_MAX_F64 ? ord : ~ord);
            } else if (t.op == DAMPR_OP_SUM_I64) {
                atomicAdd(&t.counts[slot], (u64)v);
            } else {
                const u64 ord = (u64)v ^ 0x8000000000000000ULL;
                atomicMax(&t.counts[slot], t.op == DAMPR_OP_MAX_I64 ? ord : ~ord);
            }
            if (rep == ~0ULL) return true;
            const u64 old = atomicMin(&t.reps[slot], rep);
            if (old == ~0ULL || old == rep) return true;
            if constexpr (LINE_REP) {
                *other = old;
                return true;
            }
            const u32 len = (u32)(rep & 0xFFFFFu);
            if ((u32)(old & 0xFFFFFu) != len) return false;
            const u8 *a = text + (rep >> 20), *b = text + (old >> 20);
            for (u32 i = 0; i < len; ++i)
                if (a[i] != b[i]) return false;
            return true;
        }
        slot = (slot + 1) & t.mask;
    }
    flags |= DAMPR_TF_TABLEFULL;
    return true;
}

__device__ __forceinline__ void put_record(const RecView &rv, u64 ix, u64 code, u64 bits, u32 &flags) {
    if (ix < rv.cap) rv.rec[ix] = make_ulonglong2(code, bits);
    else flags |= DAMPR_TF_RECFULL;
}

// an expression scan's key and value of a line that passed its predicates (every field bound found): the load slots
// parsed, then the programs run, or the spec's key and value read as the plain scan reads them (g0: the global offset
// of window position 0). false when the line is the host's: a missing slot field (IndexError), a slot the device does
// not parse, or a program that does not reach CPython's result.
template <int VK>
__device__ __forceinline__ bool expr_line(const u8 *t, const TupleBounds<true> &kb, const TupleView &tv,
                                          const ExprView &ex, bool kx, bool vx, int nf, const FieldsView &tab, u32 ks,
                                          u32 ke, u32 vs, u32 ve, u64 g0, long long &val, u64 &code, u64 &rep,
                                          u64 &acc_long, u32 &flags) {
    if (kb.missing) return false;
    long long lv[T_MAX];
#pragma unroll
    for (int j = 0; j < T_MAX; ++j) {
        lv[j] = 0;
        if (j < tv.n) {
            const u8 *p = t + kb.cs[j];
            const u32 len = kb.ce[j] - kb.cs[j];
            if (ex.load_kind[j] == DAMPR_LOAD_LEN) {
                lv[j] = len;
            } else if (ex.load_kind[j] == DAMPR_LOAD_INT) {
                if (!parse_int(p, len, lv[j])) return false;
            } else {
                double d;
                if (!parse_f64(p, len, d)) return false;
                lv[j] = as_i(d);
            }
        }
    }
    if (vx) {
        if (!eval_expr(ex, ex.val_prog, ex.val_len, lv[0], lv[1], lv[2], lv[3], nf, val)) return false;
    } else if constexpr (VK == VK_F64) {
        double d;
        if (!parse_f64(t + vs, ve - vs, d)) return false;
        val = as_i(d);
    } else if (tab.val_field != DAMPR_FIELD_VAL_ONE) {
        if (!parse_int(t + vs, ve - vs, val)) return false;
    }
    if (kx) {   // INT64_MIN would code to 0, the empty slot
        long long k;
        if (!eval_expr(ex, ex.key_prog, ex.key_len, lv[0], lv[1], lv[2], lv[3], nf, k) || k == X_I64_MIN) return false;
        code = (u64)k ^ 0x8000000000000000ULL;
    } else if (tab.key_int) {
        long long k;
        if (!parse_int(t + ks, ke - ks, k)) return false;
        code = (u64)k ^ 0x8000000000000000ULL;
    } else {
        const u32 klen = ke - ks;
        if (klen >= 1 && klen <= 9) {
            for (int i = (int)klen - 1; i >= 0; --i) code = (code << 7) | t[ks + i];
        } else {
            code = hash_bytes(t + ks, klen, tab.seed);
            rep = ((g0 + ks) << 20) | klen;
            acc_long++;
        }
    }
    if (VK == VK_F64 && vx && isnan(as_f(val))) flags |= DAMPR_TF_NAN;
    return true;
}

// lines per tile -> record index of each tile's first line (exclusive scan from the running count, which
// advances by the range's lines): one CTA, no inter-CTA waiting
__global__ void __launch_bounds__(SCAN_THREADS) fields_tile_scan_kernel(u64 *tiles, u64 ntiles, u64 *run) {
    __shared__ u64 warp_tot[SCAN_THREADS / 32];
    __shared__ u64 carry;
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = *run;
    __syncthreads();
    for (u64 b = 0; b < ntiles; b += SCAN_THREADS) {
        const u64 i = b + tid;
        const u64 c = i < ntiles ? tiles[i] : 0;
        u64 v = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u64 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
            if ((int)lane >= d) v += o;
        }
        if (lane == 31) warp_tot[warp] = v;
        __syncthreads();
        if (warp == 0) {
            const u64 t = warp_tot[lane];
            u64 x = t;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const u64 o = __shfl_up_sync(0xFFFFFFFFu, x, d);
                if ((int)lane >= d) x += o;
            }
            warp_tot[lane] = x - t;   // exclusive
        }
        __syncthreads();
        if (i < ntiles) tiles[i] = carry + warp_tot[warp] + v - c;
        __syncthreads();
        if (tid == SCAN_THREADS - 1) carry += warp_tot[warp] + v;
        __syncthreads();
    }
    if (tid == 0) *run = carry;
}

// a JSON scan's work on one line after pass 1 (t[q, end) is ASCII and ends at its '\n'): validate it, evaluate the
// predicates on its members, then read the key and the value. Sets to_host, dropped, val, code and rep as the field
// path does (g0: the global offset of window position 0). A kept line's key and value kinds are both reported before
// either decides that the line is the host's. JV: JsonView (top-level members) or JsonPathView (paths).
template <int VK, bool WHERE, class JV>
__device__ __forceinline__ void json_fold(const u8 *t, u32 q, u32 end, u64 g0, const FieldsView &tab,
                                          const JV &jv, const WhereView *where, bool &to_host, bool &dropped,
                                          long long &val, u64 &code, u64 &rep, u64 &acc_long, u32 &flags) {
    constexpr bool PATHS = std::is_same<JV, JsonPathView>::value;
    constexpr int JM = WHERE ? J_MAX : 2;   // the plain scan reads the key and the value only
    u32 mb[JM];
#pragma unroll
    for (int j = 0; j < JM; ++j) mb[j] = 0;
    u32 mt = 0;
    u32 bad = 0;   // PATHS: the members with a missing or non-object node above them
    bool valid;
    if constexpr (PATHS) valid = json_path_line<JM>(t, q, end, jv, mb, mt, bad);
    else valid = json_line<JM>(t, q, end, jv, mb, mt);
    if (!valid) {
        to_host = true;
        return;
    }
    if constexpr (WHERE) {
        const WhereView &wh = *where;
        const WhereProg *prog = &reinterpret_cast<const Where *>(where)->g;
        int verdict = 1;
        u32 lt = 0, lu = 0;   // a program's leaf results: T / U bits
#pragma unroll
        for (int j = 0; j < P_MAX; ++j) {
            if (j < wh.n && (verdict == 1 || prog->np)) {
                const PredSlot &pr = wh.p[j];
                const u32 ty = (mt >> (4 * pr.field)) & 0xFu;
                int r;
                if (pr.kind == DAMPR_PRED_MEMBER) {
                    r = (ty != JT_NONE) == (pr.cmp == DAMPR_CMP_IN);
                    if constexpr (PATHS) {
                        if ((bad >> pr.field) & 1u) {   // "m" in x where x is not a present object
                            r = -1;
                            const int pl = jv.up_leaf[pr.field];
                            if (pr.n == 1 && pl >= 0 && ((mt >> (4 * pl)) & 0xFu) == JT_STR) {   // x is a str
                                const u32 b = member_bounds<JM>(mb, pl);
                                const long long k = wh.c[pr.first];
                                r = contains(t + (b & 0xFFFFu), (b >> 16) - (b & 0xFFFFu), wh.b + (k >> 32), (u32)k) ==
                                    (pr.cmp == DAMPR_CMP_IN);
                            }
                        }
                    }
                } else {
                    // a member of another type than the constant's, or a missing one: the host's filter decides
                    const bool has = pr.kind == DAMPR_PRED_INT ? ty == JT_INT
                                     : pr.kind == DAMPR_PRED_F64 ? (ty == JT_INT || ty == JT_FLOAT)
                                                                 : ty == JT_STR;
                    const u32 b = member_bounds<JM>(mb, pr.field);
                    r = eval_pred(wh, pr, has, t + (b & 0xFFFFu), (b >> 16) - (b & 0xFFFFu), 0);
                }
                if (prog->np) {
                    lt |= (u32)(r == 1) << j;
                    lu |= (u32)(r < 0) << j;
                } else {
                    verdict = r;
                }
            }
        }
        if (prog->np) verdict = where_program(*prog, lt, lu);
        dropped = verdict == 0;
        to_host = verdict < 0;
        if (verdict != 1) return;
    }
    const u32 kt = (mt >> (4 * tab.key_field)) & 0xFu;
    const u32 kb = member_bounds<JM>(mb, tab.key_field);
    const u32 ks = kb & 0xFFFFu, klen = (kb >> 16) - ks;
    bool ok;   // a missing member is a KeyError in Python: the host raises it
    if (tab.key_int) {
        long long kv;
        ok = kt == JT_INT && parse_int(t + ks, klen, kv);
        if (ok) code = (u64)kv ^ 0x8000000000000000ULL;
        if (kt != JT_INT && kt != JT_NONE) flags |= DAMPR_TF_JSON_KEY_KIND;
    } else {
        ok = kt == JT_STR;   // a string with escapes is still a str: the host decodes it
        if (kt != JT_STR && kt != JT_ESC && kt != JT_NONE) flags |= DAMPR_TF_JSON_KEY_KIND;
    }
    if (tab.val_field != DAMPR_FIELD_VAL_ONE) {
        const u32 vt = (mt >> (4 * tab.val_field)) & 0xFu;
        const u32 vb = member_bounds<JM>(mb, tab.val_field);
        const u8 *vp = t + (vb & 0xFFFFu);
        const u32 vlen = (vb >> 16) - (vb & 0xFFFFu);
        if constexpr (VK == VK_F64) {
            double d;
            long long iv;
            if (vt != JT_FLOAT && vt != JT_NONE) flags |= DAMPR_TF_JSON_VAL_KIND;
            if (vt == JT_INT && parse_int(vp, vlen, iv)) val = __double_as_longlong((double)iv);   // float(-0) is 0.0
            else if ((vt == JT_INT || vt == JT_FLOAT) && parse_f64(vp, vlen, d)) val = __double_as_longlong(d);
            else ok = false;
        } else {
            if (vt != JT_INT && vt != JT_NONE) flags |= DAMPR_TF_JSON_VAL_KIND;
            if (!(vt == JT_INT && parse_int(vp, vlen, val))) ok = false;
        }
    }
    if (!ok) {
        to_host = true;
        return;
    }
    if (!tab.key_int) {
        if (klen >= 1 && klen <= 9) {
            for (int i = (int)klen - 1; i >= 0; --i) code = (code << 7) | t[ks + i];
        } else {
            code = hash_bytes(t + ks, klen, tab.seed);
            rep = ((g0 + ks) << 20) | klen;
            acc_long++;
        }
    }
}

// the kernel body over the tiles of [own_lo, own_hi); where: the predicates of a WHERE scan; WS: split on runs of
// whitespace (`line.split()`) instead of the separator byte; JSON: json.loads each line and read the members *json;
// TUP: the key is the tuple of the components that follow the predicates (where points into a TupleWhere;
// tab.key_field is component 0's field, tab.key_int is not read); EXPR: the load slots follow the predicates as TUP's
// components do, and the programs follow them (where points into an ExprWhere); JV: JsonPathView for a JSON scan
// over paths
template <int VK, int MODE, bool WHERE, bool WS, bool JSON = false, bool TUP = false, bool EXPR = false,
          class JV = JsonView>
__device__ __forceinline__ void fields_tiles(const u8 *__restrict__ text, u64 n, u64 own_lo, u64 own_hi,
                                             const FieldsView &tab, const RecView &rv, const WhereView *where,
                                             const JV *json = nullptr) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    SmemF &s = *reinterpret_cast<SmemF *>(smem_raw);
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u64 ntiles = (own_hi - own_lo + F_OWN - 1) / F_OWN;
    const bool cr_data = tab.cr_is_data != 0;
    if (tid == 0) s.flags = 0;
    if constexpr (EXPR) {   // (the first tile's __syncthreads orders this before any fold)
        HotKeys &h = hot_keys();
        if (tid < X_HOT) h.code[tid] = h.acc[tid] = 0;
    }

    u64 acc_lines = 0, acc_long = 0, acc_maxabs = 0;
    u64 acc_dropped = 0;   // WHERE: lines a predicate rejected
    u32 my_flags = 0;

    for (u64 tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const u64 sgl = own_lo + tile * (u64)F_OWN;    // global offset of window position F_LEAD
        const u32 own_len = (u32)min((u64)F_OWN, own_hi - sgl);
        const u8 *gwin = text + sgl - F_LEAD;          // global address of window position 0
        __syncthreads();                               // the previous tile's lines are done
        {
            const uint4 *src = reinterpret_cast<const uint4 *>(gwin);
            uint4 *dst = reinterpret_cast<uint4 *>(s.text);
            for (int i = tid; i < F_WIN / 16; i += F_THREADS) dst[i] = src[i];
        }
        __syncthreads();

        // ---- line starts: x in [F_LEAD, F_LEAD + own_len) with a newline at x - 1, global offset < n --------
        // thread t looks at the newlines in window bytes [F_LEAD + 64 t, +64) (starts one byte later); the start
        // at F_LEAD itself (newline at F_LEAD - 1, or the lead-in of the text) is thread 0's
        const u32 y0 = F_LEAD + 64 * tid;
        const u32 hi = F_LEAD - 1 + own_len;        // newline positions y < hi give owned starts
        u64 m = 0;
        if (y0 < hi) {
            const u32 *wp = reinterpret_cast<const u32 *>(s.text + y0);
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const u32 w = wp[i];
                const u32 nl = eq7(w & 0x7F7F7F7Fu, 0x0Au) & ~(w & 0x80808080u);
                const u32 b4 = (((nl >> 7) & 0x01010101u) * 0x01020408u) >> 24;
                m |= (u64)b4 << (4 * i);
            }
            if (y0 + 64 > hi) m &= (1ULL << (hi - y0)) - 1ULL;
            const u64 gy0 = sgl - F_LEAD + y0;      // global offset of window byte y0
            if (gy0 + 65 > n) {                     // start y0 + j + 1 must lie below n: j + 1 < n - gy0
                const u64 lim = n > gy0 ? n - gy0 : 0;
                m &= lim >= 1 ? ((1ULL << (lim - 1)) - 1ULL) : 0ULL;
            }
        }
        const bool first = tid == 0 && s.text[F_LEAD - 1] == '\n' && sgl < n;
        const u32 cnt = (u32)__popcll(m) + (first ? 1u : 0u);
        u32 v = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
            if ((int)lane >= d) v += o;
        }
        if (lane == 31) s.warp_tot[warp] = v;
        __syncthreads();
        if (warp == 0) {
            u32 t = lane < F_THREADS / 32 ? s.warp_tot[lane] : 0u;
            u32 x = t;
#pragma unroll
            for (int d = 1; d < F_THREADS / 32; d <<= 1) {
                const u32 o = __shfl_up_sync(0xFFFFFFFFu, x, d);
                if ((int)lane >= d) x += o;
            }
            if (lane < F_THREADS / 32) s.warp_tot[lane] = x - t;   // exclusive
            if (lane == F_THREADS / 32 - 1) s.nstarts = x;
        }
        __syncthreads();
        if constexpr (MODE == M_COUNT) {
            if (tid == 0) rv.tiles[tile] = s.nstarts;
            continue;
        }
        {
            u32 ix = s.warp_tot[warp] + v - cnt;
            if (first) s.starts[ix++] = (u16)F_LEAD;
            while (m) {
                const u32 j = (u32)__ffsll((long long)m) - 1u;
                m &= m - 1;
                s.starts[ix++] = (u16)(y0 + j + 1);
            }
        }
        __syncthreads();

        // ---- one line per thread -----------------------------------------------------------------------------
        const u32 nst = s.nstarts;
        const u64 tbase = MODE == M_RECORDS ? rv.tiles[tile] : 0;
        for (u32 li = tid; li < nst; li += F_THREADS) {
            const u32 q = s.starts[li];                       // window position of the first byte
            const u32 lim = min(q + (u32)F_HALO, (u32)F_WIN);  // the line's newline must lie before lim
            // pass 1: terminator, separators (WS: field starts), bytes the device does not take
            u32 p4 = q & ~3u;
            u32 nsep = 0, end = 0xFFFFFFFFu;
            bool bad = false;
            u32 skip = q & 3u;
            u32 prev = 0x80000000u;   // WS: whitespace mask of the previous 4 bytes (the byte before q is whitespace)
            for (; p4 < lim; p4 += 4) {
                const u32 w = *reinterpret_cast<const u32 *>(s.text + p4);
                u32 nl, sp, bd;
                classify<WS>(w, tab.sep, cr_data, nl, sp, bd);
                if (skip) {
                    const u32 keep = ~((1u << (8 * skip)) - 1u);
                    nl &= keep;
                    if constexpr (WS) sp |= ~keep & 0x80808080u;   // the bytes before q count as whitespace
                    else sp &= keep;
                    bd &= keep;
                    skip = 0;
                }
                if constexpr (WS) {   // field starts: non-whitespace after whitespace
                    const u32 ws = sp;
                    sp = ~ws & ((ws << 8) | (prev >> 24)) & 0x80808080u;
                    prev = ws;
                }
                if (nl) {
                    const u32 b = ((u32)__ffs(nl) - 1u) >> 3;
                    const u32 before = b ? ((1u << (8 * b)) - 1u) : 0u;
                    nsep += (u32)__popc(sp & before);
                    bad |= (bd & before) != 0;
                    end = p4 + b;
                    break;
                }
                nsep += (u32)__popc(sp);
                bad |= bd != 0;
            }
            if (end >= lim) end = 0xFFFFFFFFu;   // the newline is at or past lim: not handled here
            const u64 gq = sgl - F_LEAD + q;     // global offset of the line
            bool to_host = bad || end == 0xFFFFFFFFu;
            bool dropped = false;   // WHERE: a predicate is false
            long long val = 1, kval = 0;
            u64 code = 0, rep = ~0ULL;
            TupleBounds<TUP || EXPR> kb;   // TUP: the key components' fields and bounds; EXPR: the load slots'
            const TupleView *tup = TUP || EXPR ? &reinterpret_cast<const TupleWhere *>(where)->tup : nullptr;
            const ExprView *ex = EXPR ? &reinterpret_cast<const ExprWhere *>(where)->ex : nullptr;
            const bool kx = EXPR && ex->key_len > 0, vx = EXPR && ex->val_len > 0;   // a computed key / value
            if constexpr (JSON) {
                if (!to_host) json_fold<VK, WHERE>(s.text, q, end, gq - q, tab, *json, where, to_host, dropped, val, code,
                                                   rep, acc_long, my_flags);
            } else if (!to_host) {
                // resolve the field indices (Python semantics: negative counts from the end)
                const int nf = WS ? (int)nsep : (int)nsep + 1;
                const int ki = kx ? 0 : tab.key_field < 0 ? tab.key_field + nf : tab.key_field;
                const bool one = vx || tab.val_field == DAMPR_FIELD_VAL_ONE;
                const int vi = one ? 0 : (tab.val_field < 0 ? tab.val_field + nf : tab.val_field);
                const bool kv_missing = EXPR ? (!kx && (ki < 0 || ki >= nf)) || (!one && (vi < 0 || vi >= nf))
                                             : ki < 0 || ki >= nf || vi < 0 || vi >= nf;
                if constexpr (TUP || EXPR) {   // (tab.key_field is component 0's field: kv_missing covers it)
#pragma unroll
                    for (int j = 0; j < T_MAX; ++j) {
                        int i = -1;
                        if (j < tup->n) {
                            i = tup->field[j] < 0 ? tup->field[j] + nf : tup->field[j];
                            if (i < 0 || i >= nf) {
                                kb.missing = true;
                                i = -1;
                            }
                        }
                        kb.ci[j] = i;
                        kb.cs[j] = !WS && i == 0 ? q : 0xFFFFFFFFu;
                        kb.ce[j] = i >= 0 && i == nf - 1 ? end : 0xFFFFFFFFu;
                    }
                }
                if (!WHERE && kv_missing) {
                    to_host = true;   // IndexError: Python raises it
                } else {
                    // pass 2: field bounds (a separator at window position p closes field f and opens f + 1; WS:
                    // every field opens at a class change, the last one may run to the line end)
                    u32 ks = (!WS && ki == 0) ? q : 0xFFFFFFFFu, ke = (ki == nf - 1) ? end : 0xFFFFFFFFu;
                    u32 vs = (!WS && vi == 0) ? q : 0xFFFFFFFFu, ve = (vi == nf - 1) ? end : 0xFFFFFFFFu;
                    int need = max(ki, vi) + 1;   // separators to visit
                    // WHERE: predicate j's field is pi[j] (-1: none, IndexError in Python; -2: the whole line, which
                    // takes no bound slot), its bounds [ps[j], pe[j])
                    int pi[WHERE ? P_MAX : 1];
                    u32 ps[WHERE ? P_MAX : 1], pe[WHERE ? P_MAX : 1];
                    if constexpr (WHERE) {
                        const WhereView &wh = *where;
#pragma unroll
                        for (int j = 0; j < P_MAX; ++j) {
                            int i = -1;
                            const bool line = j < wh.n && wh.p[j].field == DAMPR_FIELD_LINE;
                            if (j < wh.n && wh.p[j].kind != DAMPR_PRED_NFIELDS && !line) {
                                i = wh.p[j].field < 0 ? wh.p[j].field + nf : wh.p[j].field;
                                if (i >= nf) i = -1;
                            }
                            pi[j] = line ? -2 : i < 0 ? -1 : i;
                            ps[j] = line || (!WS && pi[j] == 0) ? q : 0xFFFFFFFFu;
                            pe[j] = line || pi[j] == nf - 1 ? end : 0xFFFFFFFFu;
                            need = max(need, pi[j] + 1);
                        }
                    }
                    if constexpr (TUP || EXPR) {
#pragma unroll
                        for (int j = 0; j < T_MAX; ++j) need = max(need, kb.ci[j] + 1);
                    }
                    int f = 0;
                    skip = q & 3u;
                    if constexpr (WS) {
                        // f counts class changes: change 2i opens field i (its first byte), 2i + 1 closes it (the
                        // whitespace byte after it)
                        prev = 0x80000000u;
                        for (p4 = q & ~3u; f < 2 * need && p4 < end; p4 += 4) {
                            const u32 w = *reinterpret_cast<const u32 *>(s.text + p4);
                            u32 nl, ws, bd;
                            classify<true>(w, tab.sep, cr_data, nl, ws, bd);
                            if (skip) {
                                ws |= ((1u << (8 * skip)) - 1u) & 0x80808080u;
                                skip = 0;
                            }
                            u32 ch = (ws ^ ((ws << 8) | (prev >> 24))) & 0x80808080u;
                            prev = ws;
                            while (ch && f < 2 * need) {
                                const u32 p = p4 + (((u32)__ffs(ch) - 1u) >> 3);
                                ch &= ch - 1;
                                if (p >= end) break;
                                const int fi = f >> 1;
                                if (f & 1) {
                                    if (fi == ki) ke = p;
                                    if (fi == vi) ve = p;
                                    if constexpr (WHERE) {
#pragma unroll
                                        for (int j = 0; j < P_MAX; ++j)
                                            if (fi == pi[j]) pe[j] = p;
                                    }
                                    if constexpr (TUP || EXPR) {
#pragma unroll
                                        for (int j = 0; j < T_MAX; ++j)
                                            if (fi == kb.ci[j]) kb.ce[j] = p;
                                    }
                                } else {
                                    if (fi == ki) ks = p;
                                    if (fi == vi) vs = p;
                                    if constexpr (WHERE) {
#pragma unroll
                                        for (int j = 0; j < P_MAX; ++j)
                                            if (fi == pi[j]) ps[j] = p;
                                    }
                                    if constexpr (TUP || EXPR) {
#pragma unroll
                                        for (int j = 0; j < T_MAX; ++j)
                                            if (fi == kb.ci[j]) kb.cs[j] = p;
                                    }
                                }
                                ++f;
                            }
                        }
                    } else {
                        for (p4 = q & ~3u; f < need && p4 < end; p4 += 4) {
                            const u32 w = *reinterpret_cast<const u32 *>(s.text + p4);
                            u32 nl, sp, bd;
                            classify<false>(w, tab.sep, cr_data, nl, sp, bd);
                            if (skip) {
                                sp &= ~((1u << (8 * skip)) - 1u);
                                skip = 0;
                            }
                            while (sp && f < need) {
                                const u32 p = p4 + (((u32)__ffs(sp) - 1u) >> 3);
                                sp &= sp - 1;
                                if (p >= end) break;
                                if (f == ki) ke = p;
                                if (f == vi) ve = p;
                                if constexpr (WHERE) {
#pragma unroll
                                    for (int j = 0; j < P_MAX; ++j)
                                        if (f == pi[j]) pe[j] = p;
                                }
                                if constexpr (TUP || EXPR) {
#pragma unroll
                                    for (int j = 0; j < T_MAX; ++j)
                                        if (f == kb.ci[j]) kb.ce[j] = p;
                                }
                                ++f;
                                if (f == ki) ks = p + 1;
                                if (f == vi) vs = p + 1;
                                if constexpr (WHERE) {
#pragma unroll
                                    for (int j = 0; j < P_MAX; ++j)
                                        if (f == pi[j]) ps[j] = p + 1;
                                }
                                if constexpr (TUP || EXPR) {
#pragma unroll
                                    for (int j = 0; j < T_MAX; ++j)
                                        if (f == kb.ci[j]) kb.cs[j] = p + 1;
                                }
                            }
                        }
                    }
                    if constexpr (WHERE) {
                        // chain order: the first false predicate drops the line, the first undecided one (and a
                        // missing key or value field behind predicates that all hold) is the host's
                        // (a program evaluates every leaf, then folds their results)
                        const WhereView &wh = *where;
                        const WhereProg *prog = EXPR ? &reinterpret_cast<const ExprWhere *>(where)->prog
                                                : TUP ? &reinterpret_cast<const TupleWhere *>(where)->prog
                                                      : &reinterpret_cast<const Where *>(where)->g;
                        int verdict = 1;
                        u32 lt = 0, lu = 0;
#pragma unroll
                        for (int j = 0; j < P_MAX; ++j) {
                            if (j < wh.n && (verdict == 1 || prog->np)) {
                                const int r = eval_pred(wh, wh.p[j], pi[j] != -1, s.text + ps[j], pe[j] - ps[j], nf);
                                if (prog->np) {
                                    lt |= (u32)(r == 1) << j;
                                    lu |= (u32)(r < 0) << j;
                                } else {
                                    verdict = r;
                                }
                            }
                        }
                        if (prog->np) verdict = where_program(*prog, lt, lu);
                        dropped = verdict == 0;
                        to_host = verdict < 0 || (verdict == 1 && kv_missing);
                    }
                    if constexpr (EXPR) {
                        if (!WHERE || !(to_host || dropped))
                            to_host = !expr_line<VK>(s.text, kb, *tup, *ex, kx, vx, nf, tab, ks, ke, vs, ve,
                                                     sgl - F_LEAD, val, code, rep, acc_long, my_flags);
                    } else if (!WHERE || !(to_host || dropped)) {
                        const u32 klen = ke - ks;
                        if constexpr (VK == VK_F64) {
                            double d;
                            if (parse_f64(s.text + vs, ve - vs, d)) val = __double_as_longlong(d);
                            else to_host = true;
                        } else if (!one && !parse_int(s.text + vs, ve - vs, val)) {
                            to_host = true;
                        }
                        if (!to_host) {
                            if constexpr (TUP) {
                                // a missing component other than the first is an IndexError: Python raises it
                                if (!kb.missing && tuple_code(s.text, kb.cs, kb.ce, *tup, tab.seed, code))
                                    rep = (gq << 20) | (end - q);
                                else
                                    to_host = true;
                            } else if (tab.key_int) {
                                if (!parse_int(s.text + ks, klen, kval)) to_host = true;
                                else code = (u64)kval ^ 0x8000000000000000ULL;
                            } else if (klen >= 1 && klen <= 9) {
                                for (int i = (int)klen - 1; i >= 0; --i) code = (code << 7) | s.text[ks + i];
                            } else {
                                code = hash_bytes(s.text + ks, klen, tab.seed);
                                rep = ((sgl - F_LEAD + ks) << 20) | klen;
                                acc_long++;
                            }
                        }
                    }
                }
            }
            if constexpr (WHERE) {
                if (dropped) {   // the host's filters would drop it too: it goes nowhere
                    acc_dropped++;
                    if constexpr (MODE == M_RECORDS) put_record(rv, tbase + li, 0, 0, my_flags);   // a hole
                    continue;
                }
            }
            if (to_host) {
                // the host runs the stage's own functions on this line; a line longer than the device window is
                // measured here (bytes up to own_hi + 64 KB are uploaded), one of 64 KB or more ends the scan
                u32 len;
                if (end != 0xFFFFFFFFu) {
                    len = end - q;
                } else {
                    const u8 *g = text + gq;
                    len = 0;
                    while (len <= F_FB_MAXLEN && g[len] != '\n') ++len;
                }
                if (len > F_FB_MAXLEN) {
                    my_flags |= DAMPR_TF_LONGLINE;
                } else {
                    const u64 ix = atomicAdd(&tab.stats[S_FALLBACK], 1ULL);
                    if (ix < (u64)tab.fb_cap) tab.fb[ix] = (gq << 16) | (u64)len;
                    else my_flags |= DAMPR_TF_NONASCII;
                }
                if constexpr (MODE == M_RECORDS) put_record(rv, tbase + li, 0, 0, my_flags);   // a hole
                continue;
            }
            acc_lines++;
            if constexpr (VK == VK_INT) {
                const u64 av = (u64)(val < 0 ? -val : val);
                acc_maxabs = av > acc_maxabs ? av : acc_maxabs;
            } else if ((u64)val == 0x8000000000000000ULL) {
                my_flags |= DAMPR_TF_NEGZERO;
            }
            bool same;
            if constexpr (EXPR) {
                // an int-expression key folds into the CTA's hot-key slots first (a constant key, or a few buckets,
                // would otherwise send every line to one table slot); str keys keep one insert per line
                if constexpr (MODE == M_RECORDS) put_record(rv, tbase + li, code, (u64)val, my_flags);
                if (kx) {
                    HotKeys &h = hot_keys();
                    const u32 hs = (u32)mix64(code) & (X_HOT - 1);
                    const u64 c = atomicCAS(&h.code[hs], 0ULL, code);
                    const long long v = MODE == M_RECORDS ? 1 : val;
                    if (c == 0 || c == code) fold_code(&h.acc[hs], tab.op, table_code(tab.op, v));
                    else fold_insert<MODE != M_RECORDS && VK == VK_F64>(tab, text, code, v, rep, my_flags);
                    same = true;
                } else if constexpr (MODE == M_RECORDS) {
                    same = fold_insert<false>(tab, text, code, 1, rep, my_flags);
                } else {
                    same = fold_insert<VK == VK_F64>(tab, text, code, val, rep, my_flags);
                }
            } else if constexpr (TUP) {
                // the guard re-splits the entry's representative line when it is another one than this line
                u64 other = ~0ULL;
                if constexpr (MODE == M_RECORDS) {
                    put_record(rv, tbase + li, code, (u64)val, my_flags);
                    same = fold_insert<false, true>(tab, text, code, 1, rep, my_flags, &other);
                } else {
                    same = fold_insert<VK == VK_F64, true>(tab, text, code, val, rep, my_flags, &other);
                }
                if (other != ~0ULL) same = same_tuple<WS>(text, other, s.text, kb.cs, kb.ce, *tup, tab.sep);
            } else if constexpr (MODE == M_RECORDS) {
                put_record(rv, tbase + li, code, (u64)val, my_flags);
                same = fold_insert<false>(tab, text, code, 1, rep, my_flags);   // the line count of the key
            } else {
                same = fold_insert<VK == VK_F64>(tab, text, code, val, rep, my_flags);
            }
            if (!same) my_flags |= DAMPR_TF_COLLISION;
        }
    }

    if constexpr (EXPR) {   // the hot-key slots into the table, one insert per slot
        __syncthreads();
        HotKeys &h = hot_keys();
        if (tid < X_HOT && h.code[tid]) table_fold_code(tab, h.code[tid], h.acc[tid], my_flags);
    }

    // ---- publish counters ---------------------------------------------------------------------------------
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        acc_lines += __shfl_down_sync(0xFFFFFFFFu, acc_lines, d);
        acc_long += __shfl_down_sync(0xFFFFFFFFu, acc_long, d);
        const u64 o = __shfl_down_sync(0xFFFFFFFFu, acc_maxabs, d);
        acc_maxabs = o > acc_maxabs ? o : acc_maxabs;
    }
    if (lane == 0) {
        if (acc_lines) {
            atomicAdd(&tab.stats[S_LINES], acc_lines);
            atomicAdd(&tab.stats[S_FOLDED], acc_lines);
        }
        if (acc_long) atomicAdd(&tab.stats[S_LONG], acc_long);
        if (acc_maxabs) atomicMax(&tab.stats[S_MAXABS], acc_maxabs);
    }
    if constexpr (WHERE && MODE == M_TABLE) {   // record mode: records - folded - fallback
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) acc_dropped += __shfl_down_sync(0xFFFFFFFFu, acc_dropped, d);
        if (lane == 0 && acc_dropped) atomicAdd(&tab.stats[S_DROPPED], acc_dropped);
    }
    if (my_flags) atomicOr(&s.flags, my_flags);
    __syncthreads();
    if (tid == 0 && s.flags) atomicOr(&tab.stats[S_FLAGS], (u64)s.flags);
}

// the plain scan (WHERE false) and the WHERE scan, whose predicates are read in place from the parameters; WS: the
// `line.split()` build
template <int VK, int MODE, bool WHERE, bool WS>
__global__ void __launch_bounds__(F_THREADS)
text_fields_kernel(const u8 *__restrict__ text, u64 n, u64 own_lo, u64 own_hi, FieldsView tab, RecView rv) {
    static_assert(!WHERE, "a WHERE scan takes its predicates");
    static_assert(!WS || MODE != M_COUNT, "the count pass only looks at line starts");
    fields_tiles<VK, MODE, false, WS>(text, n, own_lo, own_hi, tab, rv, nullptr);
}

template <int VK, int MODE, bool WHERE, bool WS>
__global__ void __launch_bounds__(F_THREADS)
text_fields_kernel(const u8 *__restrict__ text, u64 n, u64 own_lo, u64 own_hi, FieldsView tab, RecView rv,
                   const __grid_constant__ Where where) {
    static_assert(WHERE, "a plain scan takes no predicates");
    fields_tiles<VK, MODE, true, WS>(text, n, own_lo, own_hi, tab, rv, &where.v);
}

// the JSON-lines builds: the member names (and a WHERE scan's predicates) read in place from the parameters. The
// launch runs 4 CTAs per SM; saying so keeps ptxas from squeezing the plain build into 32 registers and spilling.
template <int VK, int MODE>
__global__ void __launch_bounds__(F_THREADS, 4)
text_json_fields_kernel(const u8 *__restrict__ text, u64 n, u64 own_lo, u64 own_hi, FieldsView tab, RecView rv,
                        const __grid_constant__ JsonView json) {
    fields_tiles<VK, MODE, false, false, true>(text, n, own_lo, own_hi, tab, rv, nullptr, &json);
}

template <int VK, int MODE>
__global__ void __launch_bounds__(F_THREADS, 4)
text_json_fields_kernel(const u8 *__restrict__ text, u64 n, u64 own_lo, u64 own_hi, FieldsView tab, RecView rv,
                        const __grid_constant__ JsonView json, const __grid_constant__ Where where) {
    fields_tiles<VK, MODE, true, false, true>(text, n, own_lo, own_hi, tab, rv, &where.v, &json);
}
static_assert(sizeof(Where) + sizeof(JsonView) + 256 <= 4096, "kernel parameters");

// the JSON-lines builds over paths: the trie (and a WHERE scan's predicates) read in place from the parameters
template <int VK, int MODE>
__global__ void __launch_bounds__(F_THREADS, 4)
text_json_path_fields_kernel(const u8 *__restrict__ text, u64 n, u64 own_lo, u64 own_hi, FieldsView tab, RecView rv,
                             const __grid_constant__ JsonPathView json) {
    fields_tiles<VK, MODE, false, false, true, false, false, JsonPathView>(text, n, own_lo, own_hi, tab, rv, nullptr,
                                                                           &json);
}

template <int VK, int MODE>
__global__ void __launch_bounds__(F_THREADS, 4)
text_json_path_fields_kernel(const u8 *__restrict__ text, u64 n, u64 own_lo, u64 own_hi, FieldsView tab, RecView rv,
                             const __grid_constant__ JsonPathView json, const __grid_constant__ Where where) {
    fields_tiles<VK, MODE, true, false, true, false, false, JsonPathView>(text, n, own_lo, own_hi, tab, rv, &where.v,
                                                                          &json);
}
static_assert(sizeof(Where) + sizeof(JsonPathView) + 256 <= 4096, "kernel parameters");

// the tuple-key builds (plain and WHERE) of the separator-byte and whitespace scans: the components (and the
// predicates, unused by a plain build) read in place from the parameters. As for the JSON builds, saying that the
// plain builds run 4 CTAs per SM keeps ptxas from squeezing them into 40 registers and spilling.
template <int VK, int MODE, bool WHERE, bool WS>
__global__ void __launch_bounds__(F_THREADS, WHERE ? 1 : 4)
text_fields_tuple_kernel(const u8 *__restrict__ text, u64 n, u64 own_lo, u64 own_hi, FieldsView tab, RecView rv,
                         const __grid_constant__ TupleWhere tw) {
    static_assert(MODE != M_COUNT, "the count pass is the plain kernel's");
    fields_tiles<VK, MODE, WHERE, WS, false, true>(text, n, own_lo, own_hi, tab, rv, &tw.where);
}
static_assert(sizeof(TupleWhere) + 256 <= 4096, "kernel parameters");

// the expression builds (plain and WHERE) of the separator-byte and whitespace scans: the load slots, the programs
// (and the predicates, unused by a plain build) read in place from the parameters
template <int VK, int MODE, bool WHERE, bool WS>
__global__ void __launch_bounds__(F_THREADS, 4)
text_fields_expr_kernel(const u8 *__restrict__ text, u64 n, u64 own_lo, u64 own_hi, FieldsView tab, RecView rv,
                        const __grid_constant__ ExprWhere xw) {
    static_assert(MODE != M_COUNT, "the count pass is the plain kernel's");
    fields_tiles<VK, MODE, WHERE, WS, false, false, true>(text, n, own_lo, own_hi, tab, rv, &xw.where);
}
static_assert(sizeof(ExprWhere) + 256 <= 4096, "kernel parameters");

// one kernel over the tiles of [own_lo, own_hi); WHERE: the build that applies the predicates *wh; WS: the
// whitespace-split build; JSON: the JSON-lines build over the members *jv; TUP: the tuple-key build over *tk; xe: the
// expression build over the load slots *tk and the programs *xe; pv: the JSON build over the member paths *pv
template <int VK, int MODE, bool WHERE = false, bool WS = false, bool JSON = false, bool TUP = false>
int launch_fields(dampr_ctx *ctx, dampr_textbuf *tb, u64 own_lo, u64 own_hi, const FieldsView &tv, const RecView &rv,
                  int timer, const Where *wh = nullptr, const JsonView *jv = nullptr,
                  const TupleView *tk = nullptr, const ExprView *xe = nullptr, const JsonPathView *pv = nullptr) {
    const size_t smem = sizeof(SmemF);
    const u64 ntiles = (own_hi - own_lo + F_OWN - 1) / F_OWN;
    u64 grid = (u64)ctx->num_sms * 4;
    if (grid > ntiles) grid = ntiles;
    if (xe) {
        if constexpr (!JSON && !TUP && MODE != M_COUNT) {
            ExprWhere xw{};
            if (wh) {
                xw.where = wh->v;
                xw.prog = wh->g;
            }
            xw.tup = *tk;
            xw.ex = *xe;
            void (*kernel)(const u8 *, u64, u64, u64, FieldsView, RecView, ExprWhere) =
                text_fields_expr_kernel<VK, MODE, WHERE, WS>;
            CUDA_TRY(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ScopedTimer tm(ctx, timer);
            kernel<<<(unsigned)grid, F_THREADS, smem, ctx->stream>>>(tb->text, tb->n, own_lo, own_hi, tv, rv, xw);
        }
    } else if constexpr (TUP) {
        TupleWhere tw{};
        if (wh) {
            tw.where = wh->v;
            tw.prog = wh->g;
        }
        tw.tup = *tk;
        void (*kernel)(const u8 *, u64, u64, u64, FieldsView, RecView, TupleWhere) =
            text_fields_tuple_kernel<VK, MODE, WHERE, WS>;
        CUDA_TRY(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ScopedTimer tm(ctx, timer);
        kernel<<<(unsigned)grid, F_THREADS, smem, ctx->stream>>>(tb->text, tb->n, own_lo, own_hi, tv, rv, tw);
    } else if constexpr (JSON && WHERE) {
        if (pv) {
            void (*kernel)(const u8 *, u64, u64, u64, FieldsView, RecView, JsonPathView, Where) =
                text_json_path_fields_kernel<VK, MODE>;
            CUDA_TRY(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ScopedTimer tm(ctx, timer);
            kernel<<<(unsigned)grid, F_THREADS, smem, ctx->stream>>>(tb->text, tb->n, own_lo, own_hi, tv, rv, *pv, *wh);
        } else {
            void (*kernel)(const u8 *, u64, u64, u64, FieldsView, RecView, JsonView, Where) =
                text_json_fields_kernel<VK, MODE>;
            CUDA_TRY(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ScopedTimer tm(ctx, timer);
            kernel<<<(unsigned)grid, F_THREADS, smem, ctx->stream>>>(tb->text, tb->n, own_lo, own_hi, tv, rv, *jv, *wh);
        }
    } else if constexpr (JSON) {
        if (pv) {
            void (*kernel)(const u8 *, u64, u64, u64, FieldsView, RecView, JsonPathView) =
                text_json_path_fields_kernel<VK, MODE>;
            CUDA_TRY(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ScopedTimer tm(ctx, timer);
            kernel<<<(unsigned)grid, F_THREADS, smem, ctx->stream>>>(tb->text, tb->n, own_lo, own_hi, tv, rv, *pv);
        } else {
            void (*kernel)(const u8 *, u64, u64, u64, FieldsView, RecView, JsonView) = text_json_fields_kernel<VK, MODE>;
            CUDA_TRY(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            ScopedTimer tm(ctx, timer);
            kernel<<<(unsigned)grid, F_THREADS, smem, ctx->stream>>>(tb->text, tb->n, own_lo, own_hi, tv, rv, *jv);
        }
    } else if constexpr (WHERE) {
        void (*kernel)(const u8 *, u64, u64, u64, FieldsView, RecView, Where) =
            text_fields_kernel<VK, MODE, true, WS>;
        CUDA_TRY(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ScopedTimer tm(ctx, timer);
        kernel<<<(unsigned)grid, F_THREADS, smem, ctx->stream>>>(tb->text, tb->n, own_lo, own_hi, tv, rv, *wh);
    } else {
        void (*kernel)(const u8 *, u64, u64, u64, FieldsView, RecView) = text_fields_kernel<VK, MODE, false, WS>;
        CUDA_TRY(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ScopedTimer tm(ctx, timer);
        kernel<<<(unsigned)grid, F_THREADS, smem, ctx->stream>>>(tb->text, tb->n, own_lo, own_hi, tv, rv);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return DAMPR_OK;
}

// the predicates of spec in kernel-parameter form; DAMPR_ERR_ARG for a kind, comparison or limit outside the header's
// (json: the predicates of a JSON scan, whose fields index the nmembers members; DAMPR_PRED_MEMBER instead of NFIELDS;
// paths: a call over member paths, whose DAMPR_PRED_MEMBER may carry one STR constant)
int where_view(dampr_ctx *ctx, const dampr_fields_spec *spec, Where &wv, bool json = false, int nmembers = 0,
               bool paths = false) {
    ARG_CHECK(ctx, spec->npreds >= 0 && spec->npreds <= DAMPR_PRED_MAX + DAMPR_PRED_MAX_OPS,
              "npreds must be 0 .. DAMPR_PRED_MAX + DAMPR_PRED_MAX_OPS");
    ARG_CHECK(ctx, spec->npreds == 0 || spec->preds != nullptr, "null preds");
    wv = Where{};
    WhereView &w = wv.v;
    WhereProg &g = wv.g;
    int nc = 0, nb = 0, nops = 0, depth = 0;
    for (int e = 0; e < spec->npreds; ++e) {
        const dampr_field_pred &p = spec->preds[e];
        if (p.kind >= DAMPR_PRED_AND && p.kind <= DAMPR_PRED_NOT) {
            const int pops = p.kind == DAMPR_PRED_NOT ? 1 : 2;
            ARG_CHECK(ctx, depth >= pops, "a connective finds fewer operands than it takes");
            ARG_CHECK(ctx, p.n == 0, "a connective takes no constants");
            ARG_CHECK(ctx, ++nops <= DAMPR_PRED_MAX_OPS, "more than DAMPR_PRED_MAX_OPS connectives");
            depth -= pops - 1;
            g.op[g.np++] = (u8)(W_AND + (p.kind - DAMPR_PRED_AND));
            continue;
        }
        ARG_CHECK(ctx, w.n < DAMPR_PRED_MAX, "more than DAMPR_PRED_MAX predicates");
        const int j = w.n++;
        g.op[g.np++] = (u8)j;
        ++depth;
        const bool in = p.cmp == DAMPR_CMP_IN || p.cmp == DAMPR_CMP_NOT_IN;
        const bool member = json && p.kind == DAMPR_PRED_MEMBER;
        const bool text = p.kind == DAMPR_PRED_LEN || p.kind == DAMPR_PRED_NONBLANK;   // of a str field only
        const bool any = p.cmp == DAMPR_CMP_STARTS || p.cmp == DAMPR_CMP_ENDS;         // n constants, any match
        if (p.field == DAMPR_FIELD_LINE) {
            ARG_CHECK(ctx, !json, "a JSON scan has no line operand");
            ARG_CHECK(ctx, p.kind == DAMPR_PRED_STR || text, "the line operand is a str");
        } else if (json) {
            ARG_CHECK(ctx, p.kind >= DAMPR_PRED_STR && p.kind <= DAMPR_PRED_NONBLANK && p.kind != DAMPR_PRED_NFIELDS,
                      "predicate kind of a JSON scan");
            ARG_CHECK(ctx, p.field >= 0 && p.field < nmembers, "a JSON predicate's field must index the members");
        } else {
            ARG_CHECK(ctx, p.kind >= DAMPR_PRED_STR && p.kind <= DAMPR_PRED_NONBLANK && p.kind != DAMPR_PRED_MEMBER,
                      "predicate kind");
        }
        ARG_CHECK(ctx, p.cmp >= DAMPR_CMP_EQ && p.cmp <= DAMPR_CMP_ENDS, "predicate comparison");
        ARG_CHECK(ctx, !member || in, "DAMPR_PRED_MEMBER takes IN or NOT_IN");
        ARG_CHECK(ctx, !in || member || p.kind == DAMPR_PRED_STR || p.kind == DAMPR_PRED_INT,
                  "IN / NOT_IN take STR or INT");
        ARG_CHECK(ctx, p.cmp < DAMPR_CMP_CONTAINS || p.kind == DAMPR_PRED_STR, "CONTAINS .. ENDS take STR");
        ARG_CHECK(ctx, p.kind != DAMPR_PRED_LEN || p.cmp <= DAMPR_CMP_GE, "LEN takes EQ .. GE");
        ARG_CHECK(ctx, p.kind != DAMPR_PRED_NONBLANK || p.cmp == DAMPR_CMP_EQ, "NONBLANK takes EQ");
        ARG_CHECK(ctx, member                               ? (p.n == 0 || (paths && p.n == 1))
                       : p.kind == DAMPR_PRED_NONBLANK      ? p.n == 0
                       : in || any                          ? (p.n >= 1 && p.n <= DAMPR_PRED_MAX_CONSTS)
                                                            : p.n == 1,
                  "predicate constant count");
        ARG_CHECK(ctx, nc + p.n <= DAMPR_PRED_MAX_CONSTS, "more than DAMPR_PRED_MAX_CONSTS predicate constants");
        w.p[j] = PredSlot{p.field, (u8)p.kind, (u8)p.cmp, (u8)nc, (u8)p.n};
        for (int i = 0; i < p.n; ++i, ++nc) {
            if (p.kind == DAMPR_PRED_F64) {
                long long bits;
                memcpy(&bits, &p.f64, sizeof bits);
                w.c[nc] = bits;
            } else if (p.kind == DAMPR_PRED_STR || member) {
                ARG_CHECK(ctx, p.bytes != nullptr && p.lens != nullptr, "null predicate strings");
                ARG_CHECK(ctx, p.lens[i] <= (uint32_t)(DAMPR_PRED_MAX_BYTES - nb),
                          "more than DAMPR_PRED_MAX_BYTES bytes of predicate strings");
                u32 off = 0;
                for (int k = 0; k < i; ++k) off += p.lens[k];
                if (p.lens[i]) memcpy(w.b + nb, p.bytes + off, p.lens[i]);
                w.c[nc] = ((long long)nb << 32) | p.lens[i];
                nb += (int)p.lens[i];
            } else {
                ARG_CHECK(ctx, p.ints != nullptr, "null predicate constants");
                w.c[nc] = p.ints[i];
            }
        }
    }
    if (!nops) g.np = 0;   // no connective: the leaves are the AND chain
    return DAMPR_OK;
}

int check_fields_args(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, u64 own_lo, u64 own_hi,
                      const dampr_fields_spec *spec) {
    ARG_CHECK(ctx, ctx && t && tb && spec, "null");
    ARG_CHECK(ctx, own_lo <= own_hi && own_hi <= tb->n, "ownership range outside the text");
    ARG_CHECK(ctx, (own_lo % 16) == 0, "own_lo must be a multiple of 16");
    ARG_CHECK(ctx, spec->sep == DAMPR_FIELD_SEP_WS ||
                       (spec->sep > 0 && spec->sep < 0x80 && spec->sep != '\n' && spec->sep != '\r'),
              "separator must be DAMPR_FIELD_SEP_WS or an ASCII byte other than NUL, '\\n' and '\\r'");
    ARG_CHECK(ctx, spec->key_kind == DAMPR_FIELD_KEY_STR || spec->key_kind == DAMPR_FIELD_KEY_INT, "key kind");
    Where w;
    return where_view(ctx, spec, w);
}

// the trie of a JSON call whose members hold a path (names joined by DAMPR_JSON_PATH_SEP)
int json_path_view(dampr_ctx *ctx, const dampr_json_members *m, JsonPathView &pv) {
    pv = JsonPathView{};
    pv.n = m->n;
    for (int k = 0; k < J_NODES; ++k) pv.up[k] = pv.leaf[k] = -1;
    int nn = 0, off = 0;
    int node_of[J_MAX];
    for (int j = 0; j < m->n; ++j) {
        const int len = m->len[j];
        ARG_CHECK(ctx, len >= 0 && len < DAMPR_JSON_MAX_PATH * (J_NAME + 1),
                  "a member of 1 .. DAMPR_JSON_MAX_PATH names of 0 .. DAMPR_JSON_MAX_NAME bytes");
        const char *b = m->bytes + off;
        int names = 1;
        for (int i = 0; i < len; ++i) names += b[i] == DAMPR_JSON_PATH_SEP;
        ARG_CHECK(ctx, names <= DAMPR_JSON_MAX_PATH, "a path of more than DAMPR_JSON_MAX_PATH names");
        int parent = -1, s = 0;
        u16 anc = 0;
        for (int x = 0; x < names; ++x) {
            int e = s;
            while (e < len && b[e] != DAMPR_JSON_PATH_SEP) ++e;
            const int nl = e - s;
            ARG_CHECK(ctx, names == 1 || nl >= 1, "an empty name in a path");
            ARG_CHECK(ctx, nl <= J_NAME, "a member name of 0 .. DAMPR_JSON_MAX_NAME bytes");
            for (int i = s; i < e; ++i) {
                const u8 c = (u8)b[i];
                ARG_CHECK(ctx, c >= 0x20 && c < 0x80 && c != '"' && c != '\\',
                          "member names are ASCII without '\"', '\\\\' or bytes below 0x20");
            }
            int k = 0;
            while (k < nn && !(pv.up[k] == parent && pv.len[k] == nl && memcmp(pv.name[k], b + s, nl) == 0)) ++k;
            if (k == nn) {
                ARG_CHECK(ctx, nn < J_NODES, "more than DAMPR_JSON_MAX_NODES path nodes");
                pv.up[k] = (signed char)parent;
                pv.len[k] = (u8)nl;
                memcpy(pv.name[k], b + s, nl);
                ++nn;
            }
            if (x + 1 < names) {
                anc |= (u16)(1u << k);
                parent = k;
            } else {
                ARG_CHECK(ctx, pv.leaf[k] < 0, "two members name the same path");
                pv.leaf[k] = (signed char)j;
                pv.anc[j] = anc;
                node_of[j] = k;
            }
            s = e + 1;
        }
        off += len;
    }
    for (int j = 0; j < m->n; ++j)
        pv.up_leaf[j] = pv.up[node_of[j]] >= 0 ? pv.leaf[pv.up[node_of[j]]] : (signed char)-1;
    for (int k = 0; k < nn; ++k) {
        pv.kids[pv.up[k] + 1] |= (u16)(1u << k);
        for (int a = pv.up[k]; a >= 0; a = pv.up[a]) {
            pv.sub[a] |= (u16)(1u << k);
            if (pv.leaf[k] >= 0) pv.sub_types[a] |= 0xFu << (4 * pv.leaf[k]);
        }
    }
    return DAMPR_OK;
}

// the arguments of a JSON call in kernel-parameter form: its predicates w, and its members as the names jv, or as the
// trie pv (paths set) when a member is a path
int check_json_args(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, u64 own_lo, u64 own_hi,
                    const dampr_fields_spec *spec, const dampr_json_members *m, JsonView &jv, JsonPathView &pv,
                    bool &paths, Where &w) {
    ARG_CHECK(ctx, ctx && t && tb && spec && m, "null");
    ARG_CHECK(ctx, own_lo <= own_hi && own_hi <= tb->n, "ownership range outside the text");
    ARG_CHECK(ctx, (own_lo % 16) == 0, "own_lo must be a multiple of 16");
    ARG_CHECK(ctx, spec->sep == DAMPR_FIELD_SEP_JSON, "a JSON call takes sep DAMPR_FIELD_SEP_JSON");
    ARG_CHECK(ctx, spec->key_kind == DAMPR_FIELD_KEY_STR || spec->key_kind == DAMPR_FIELD_KEY_INT, "key kind");
    ARG_CHECK(ctx, m->n >= 1 && m->n <= J_MAX, "1 .. DAMPR_JSON_MAX_MEMBERS members");
    ARG_CHECK(ctx, m->len != nullptr && m->bytes != nullptr, "null member names");
    ARG_CHECK(ctx, spec->key_field >= 0 && spec->key_field < m->n, "key_field must index the members");
    ARG_CHECK(ctx, spec->val_field == DAMPR_FIELD_VAL_ONE || (spec->val_field >= 0 && spec->val_field < m->n),
              "val_field must index the members or be DAMPR_FIELD_VAL_ONE");
    paths = false;
    for (int j = 0, off = 0; j < m->n && m->len[j] >= 0 && m->len[j] < DAMPR_JSON_MAX_PATH * (J_NAME + 1); ++j) {
        paths |= memchr(m->bytes + off, DAMPR_JSON_PATH_SEP, m->len[j]) != nullptr;
        off += m->len[j];
    }
    if (paths) {
        if (int r = json_path_view(ctx, m, pv)) return r;
        return where_view(ctx, spec, w, true, m->n, true);
    }
    jv = JsonView{};
    jv.n = m->n;
    int off = 0;
    for (int j = 0; j < m->n; ++j) {
        ARG_CHECK(ctx, m->len[j] >= 0 && m->len[j] <= J_NAME, "a member name of 0 .. DAMPR_JSON_MAX_NAME bytes");
        for (int i = 0; i < m->len[j]; ++i) {
            const u8 c = (u8)m->bytes[off + i];
            ARG_CHECK(ctx, c >= 0x20 && c < 0x80 && c != '"' && c != '\\',
                      "member names are ASCII without '\"', '\\\\' or bytes below 0x20");
            jv.name[j][i] = c;
        }
        jv.len[j] = (u8)m->len[j];
        off += m->len[j];
    }
    return where_view(ctx, spec, w, true, m->n);
}

FieldsView fields_view(dampr_table *t, const dampr_fields_spec *spec, int op) {
    return FieldsView{t->keys, t->counts, t->reps, t->stats, t->fb, t->cap - 1, 0x243F6A8885A308D3ULL, t->fb_cap,
                      (u32)spec->sep, spec->key_field, spec->val_field, spec->key_kind == DAMPR_FIELD_KEY_INT ? 1 : 0,
                      op, spec->cr_is_data ? 1u : 0u};
}

// the fold pass of one range under one separator class: the plain kernel, or its WHERE build when spec holds
// predicates; tk: the tuple-key builds over those components; xe: the expression builds over the load slots tk
template <int VK, int MODE, bool WS>
int launch_fold_sep(dampr_ctx *ctx, dampr_textbuf *tb, u64 own_lo, u64 own_hi, const dampr_fields_spec *spec,
                    const FieldsView &tv, const RecView &rv, const TupleView *tk, const ExprView *xe = nullptr) {
    if (xe) {
        Where w{};
        if (spec->npreds == 0)
            return launch_fields<VK, MODE, false, WS>(ctx, tb, own_lo, own_hi, tv, rv, DAMPR_K_TEXT_FIELDS, nullptr,
                                                      nullptr, tk, xe);
        if (int r = where_view(ctx, spec, w)) return r;
        return launch_fields<VK, MODE, true, WS>(ctx, tb, own_lo, own_hi, tv, rv, DAMPR_K_TEXT_FIELDS, &w, nullptr,
                                                 tk, xe);
    }
    if (spec->npreds == 0) {
        if (!tk) return launch_fields<VK, MODE, false, WS>(ctx, tb, own_lo, own_hi, tv, rv, DAMPR_K_TEXT_FIELDS);
        return launch_fields<VK, MODE, false, WS, false, true>(ctx, tb, own_lo, own_hi, tv, rv, DAMPR_K_TEXT_FIELDS,
                                                               nullptr, nullptr, tk);
    }
    Where w;
    if (int r = where_view(ctx, spec, w)) return r;
    if (!tk) return launch_fields<VK, MODE, true, WS>(ctx, tb, own_lo, own_hi, tv, rv, DAMPR_K_TEXT_FIELDS, &w);
    return launch_fields<VK, MODE, true, WS, false, true>(ctx, tb, own_lo, own_hi, tv, rv, DAMPR_K_TEXT_FIELDS, &w,
                                                          nullptr, tk);
}

// the fold pass of one range of a JSON scan over the names jv, or the member paths *pv: the plain build reads two
// members, the WHERE build (also taken without predicates when more members are listed) up to J_MAX
template <int VK, int MODE>
int launch_json_fold(dampr_ctx *ctx, dampr_textbuf *tb, u64 own_lo, u64 own_hi, const dampr_fields_spec *spec,
                     const JsonView &jv, const JsonPathView *pv, const Where &w, const FieldsView &tv,
                     const RecView &rv) {
    if (spec->npreds == 0 && (pv ? pv->n : jv.n) <= 2)
        return launch_fields<VK, MODE, false, false, true>(ctx, tb, own_lo, own_hi, tv, rv, DAMPR_K_TEXT_FIELDS,
                                                          nullptr, &jv, nullptr, nullptr, pv);
    return launch_fields<VK, MODE, true, false, true>(ctx, tb, own_lo, own_hi, tv, rv, DAMPR_K_TEXT_FIELDS, &w, &jv,
                                                      nullptr, nullptr, pv);
}

// the fold pass of one range: the separator-byte build, or the whitespace-split one under DAMPR_FIELD_SEP_WS
template <int VK, int MODE>
int launch_fold(dampr_ctx *ctx, dampr_textbuf *tb, u64 own_lo, u64 own_hi, const dampr_fields_spec *spec,
                const FieldsView &tv, const RecView &rv, const TupleView *tk = nullptr, const ExprView *xe = nullptr) {
    if (spec->sep == DAMPR_FIELD_SEP_WS)
        return launch_fold_sep<VK, MODE, true>(ctx, tb, own_lo, own_hi, spec, tv, rv, tk, xe);
    return launch_fold_sep<VK, MODE, false>(ctx, tb, own_lo, own_hi, spec, tv, rv, tk, xe);
}

// the components of a tuple-key call in kernel-parameter form
int tuple_view(dampr_ctx *ctx, const dampr_field_keys *keys, TupleView &tk) {
    ARG_CHECK(ctx, keys != nullptr, "null");
    ARG_CHECK(ctx, keys->n >= 1 && keys->n <= T_MAX, "1 .. DAMPR_FIELD_KEYS_MAX key components");
    tk = TupleView{};
    tk.n = keys->n;
    for (int j = 0; j < keys->n; ++j) {
        ARG_CHECK(ctx, keys->kind[j] == DAMPR_FIELD_KEY_STR || keys->kind[j] == DAMPR_FIELD_KEY_INT,
                  "key component kind");
        tk.field[j] = keys->field[j];
        tk.is_int[j] = keys->kind[j] == DAMPR_FIELD_KEY_INT;
    }
    return DAMPR_OK;
}

// one program of an expression call, checked once: every operation finds operands of its type, the stack stays
// within X_DEPTH and ends with one value of type want ('i' or 'f'); constants and load slots (kinds lk) in range
bool expr_program_ok(const int32_t *prog, int len, char want, const int32_t *lk, int nloads) {
    if (len < 1 || len > X_OPS) return false;
    char st[X_DEPTH];
    int sp = 0;
    for (int pc = 0; pc < len; ++pc) {
        const int op = prog[pc] & 0xFF, arg = prog[pc] >> 8;
        char push = 0, in = 0, out = 0;   // a leaf's type, or an operation's operand and result types
        int arity = 0;
        switch (op) {
            case EV_CI: push = arg >= 0 && arg < X_CONSTS ? 'i' : 0; break;
            case EV_CF: push = arg >= 0 && arg < X_CONSTS ? 'f' : 0; break;
            case EV_LOAD: push = arg >= 0 && arg < nloads ? (lk[arg] == DAMPR_LOAD_F64 ? 'f' : 'i') : 0; break;
            case EV_NF: push = 'i'; break;
            case EV_I2F: arity = 1, in = 'i', out = 'f'; break;
            case EV_F2I: arity = 1, in = 'f', out = 'i'; break;
            case EV_INEG: case EV_IABS: arity = 1, in = out = 'i'; break;
            case EV_FNEG: case EV_FABS: arity = 1, in = out = 'f'; break;
            case EV_IADD: case EV_ISUB: case EV_IMUL: case EV_IFLOOR: case EV_IMOD: arity = 2, in = out = 'i'; break;
            case EV_IDIV: arity = 2, in = 'i', out = 'f'; break;
            case EV_FADD: case EV_FSUB: case EV_FMUL: case EV_FDIV: arity = 2, in = out = 'f'; break;
            default: return false;   // EV_X, EV_LOG and unknown opcodes
        }
        if (arity == 0) {
            if (!push || sp == X_DEPTH) return false;
            st[sp++] = push;
            continue;
        }
        if (sp < arity) return false;
        for (int i = 0; i < arity; ++i)
            if (st[sp - 1 - i] != in) return false;
        sp -= arity;
        st[sp++] = out;
    }
    return sp == 1 && st[0] == want;
}

// the load slots (as tuple components) and programs of an expression call in kernel-parameter form; f64: the value
// type op folds
int expr_view(dampr_ctx *ctx, const dampr_field_expr *x, bool f64, TupleView &tk, ExprView &ev) {
    ARG_CHECK(ctx, x != nullptr, "null");
    ARG_CHECK(ctx, x->nloads >= 0 && x->nloads <= DAMPR_EXPR_MAX_LOADS, "0 .. DAMPR_EXPR_MAX_LOADS load slots");
    tk = TupleView{};
    ev = ExprView{};
    tk.n = x->nloads;
    for (int j = 0; j < x->nloads; ++j) {
        ARG_CHECK(ctx, x->load_kind[j] >= DAMPR_LOAD_INT && x->load_kind[j] <= DAMPR_LOAD_LEN, "load slot kind");
        tk.field[j] = x->load_field[j];
        ev.load_kind[j] = x->load_kind[j];
    }
    ARG_CHECK(ctx, x->key_type == DAMPR_EXPR_NONE || x->key_type == DAMPR_EXPR_INT, "key_type");
    ARG_CHECK(ctx, x->val_type >= DAMPR_EXPR_NONE && x->val_type <= DAMPR_EXPR_F64, "val_type");
    ARG_CHECK(ctx, x->key_type != DAMPR_EXPR_NONE || x->val_type != DAMPR_EXPR_NONE, "no program");
    ARG_CHECK(ctx, x->val_type == DAMPR_EXPR_NONE || (x->val_type == DAMPR_EXPR_F64) == f64,
              "the value program's type must be the one op folds");
    if (x->key_type != DAMPR_EXPR_NONE) {
        ARG_CHECK(ctx, expr_program_ok(x->key_prog, x->key_len, 'i', x->load_kind, x->nloads), "malformed key program");
        ev.key_len = x->key_len;
        memcpy(ev.key_prog, x->key_prog, sizeof ev.key_prog);
    }
    if (x->val_type != DAMPR_EXPR_NONE) {
        ARG_CHECK(ctx, expr_program_ok(x->val_prog, x->val_len, f64 ? 'f' : 'i', x->load_kind, x->nloads),
                  "malformed value program");
        ev.val_len = x->val_len;
        memcpy(ev.val_prog, x->val_prog, sizeof ev.val_prog);
    }
    memcpy(ev.ci, x->ci, sizeof ev.ci);
    memcpy(ev.cf, x->cf, sizeof ev.cf);
    return DAMPR_OK;
}

// fields_view of a tuple-key call: its key field is component 0's (the scan's missing-field rule checks it with the
// value field; the tuple build checks the others)
FieldsView tuple_fields_view(dampr_table *t, const dampr_fields_spec *spec, int op, const TupleView &tk) {
    FieldsView tv = fields_view(t, spec, op);
    tv.key_field = tk.field[0];
    tv.key_int = 0;
    return tv;
}

// the columns of dampr_table_fetch_field_keys on the device
struct TupleCols {
    u8 *str[T_MAX];
    long long *ints[T_MAX];
    u32 width[T_MAX];
};

// one entry of a tuple-key table per thread: its representative line split again. maxlen != nullptr: the longest
// str component of each column only; else the entry's row (compacted through cursor) of every column
template <bool WS>
__global__ void table_tuple_keys_kernel(const u64 *__restrict__ keys, const u64 *__restrict__ counts,
                                        const u64 *__restrict__ reps, u64 cap, const u8 *__restrict__ text, u32 sep,
                                        const __grid_constant__ TupleView tv, const __grid_constant__ TupleCols out,
                                        u64 *out_counts, u64 *out_codes, u64 out_cap, u64 *cursor, u32 *maxlen) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x; i < cap; i += stride) {
        const u64 k = keys[i];
        const bool have = k != 0;
        u64 idx = 0;
        if (!maxlen) {
            const u32 m = __ballot_sync(0xFFFFFFFFu, have);
            u64 base = 0;
            if (m) {
                const int leader = __ffs(m) - 1;
                if ((int)(threadIdx.x & 31) == leader) base = atomicAdd(cursor, (u64)__popc(m));
                base = __shfl_sync(0xFFFFFFFFu, base, leader);
            }
            idx = base + __popc(m & ((1u << (threadIdx.x & 31)) - 1u));
        }
        if (!have || (!maxlen && idx >= out_cap)) continue;
        const u64 rep = reps[i];
        const u8 *p = text + (rep >> 20);
        u32 s[T_MAX], e[T_MAX];
        line_fields<WS>(p, (u32)(rep & 0xFFFFFu), sep, tv, s, e);
#pragma unroll
        for (int j = 0; j < T_MAX; ++j) {
            if (j >= tv.n) continue;
            if (maxlen) {
                if (!tv.is_int[j]) atomicMax(&maxlen[j], e[j] - s[j]);
            } else if (tv.is_int[j]) {
                long long v = 0;
                parse_int(p + s[j], e[j] - s[j], v);
                out.ints[j][idx] = v;
            } else {
                const u32 w = out.width[j], len = min(e[j] - s[j], w);
                u8 *o = out.str[j] + idx * w;
                for (u32 b = 0; b < len; ++b) o[b] = p[s[j] + b];
                for (u32 b = len; b < w; ++b) o[b] = 0;
            }
        }
        if (maxlen) continue;
        if (out_counts) out_counts[idx] = counts[i];
        if (out_codes) out_codes[idx] = k;
    }
}

// record mode's first two kernels over one range: lines per tile (the tile array grown to the range), then the
// tile bases scanned from the running record count
int count_records(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, u64 own_lo, u64 own_hi, const FieldsView &tv,
                  RecView &rv) {
    const u64 ntiles = (own_hi - own_lo + F_OWN - 1) / F_OWN;
    if (ntiles > t->tiles_cap) {
        CUDA_TRY(ctx, cudaStreamSynchronize(ctx->stream));   // the previous range may still read the old array
        cudaFree(t->tiles);
        t->tiles = nullptr;
        t->tiles_cap = 0;
        CUDA_TRY(ctx, cudaMalloc(&t->tiles, ntiles * sizeof(u64)));
        t->tiles_cap = ntiles;
    }
    rv.tiles = t->tiles;
    wait_uploads(ctx);
    if (int r = launch_fields<VK_INT, M_COUNT>(ctx, tb, own_lo, own_hi, tv, rv, DAMPR_K_TEXT_FIELDS_COUNT)) return r;
    {
        ScopedTimer tm(ctx, DAMPR_K_TEXT_FIELDS_COUNT);
        fields_tile_scan_kernel<<<1, SCAN_THREADS, 0, ctx->stream>>>(t->tiles, ntiles, t->stats + S_RECORDS);
    }
    CUDA_TRY(ctx, cudaGetLastError());
    return DAMPR_OK;
}

}  // namespace

extern "C" int32_t dampr_text_fields(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                                     uint64_t own_hi, const dampr_fields_spec *spec) {
    if (int r = check_fields_args(ctx, t, tb, own_lo, own_hi, spec)) return r;
    const bool f64 = spec->op == DAMPR_OP_MIN_F64 || spec->op == DAMPR_OP_MAX_F64;
    ARG_CHECK(ctx, f64 || spec->op == DAMPR_OP_SUM_I64 || spec->op == DAMPR_OP_MIN_I64 ||
                       spec->op == DAMPR_OP_MAX_I64,
              "op must be DAMPR_OP_SUM_I64, DAMPR_OP_MIN_I64, DAMPR_OP_MAX_I64, DAMPR_OP_MIN_F64 or DAMPR_OP_MAX_F64");
    ARG_CHECK(ctx, !f64 || spec->val_field != DAMPR_FIELD_VAL_ONE, "a float op needs a value field");
    if (own_hi <= own_lo) return DAMPR_OK;
    const FieldsView tv = fields_view(t, spec, spec->op);
    wait_uploads(ctx);
    if (f64) return launch_fold<VK_F64, M_TABLE>(ctx, tb, own_lo, own_hi, spec, tv, RecView{});
    return launch_fold<VK_INT, M_TABLE>(ctx, tb, own_lo, own_hi, spec, tv, RecView{});
}

extern "C" int32_t dampr_text_fields_records(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                                             uint64_t own_hi, const dampr_fields_spec *spec, dampr_kv *rec) {
    if (int r = check_fields_args(ctx, t, tb, own_lo, own_hi, spec)) return r;
    ARG_CHECK(ctx, rec != nullptr, "null");
    ARG_CHECK(ctx, spec->op == DAMPR_OP_SUM_I64 || spec->op == DAMPR_OP_SUM_F64,
              "op must be DAMPR_OP_SUM_I64 or DAMPR_OP_SUM_F64");
    ARG_CHECK(ctx, spec->val_field != DAMPR_FIELD_VAL_ONE, "record mode needs a value field");
    if (own_hi <= own_lo) return DAMPR_OK;
    const FieldsView tv = fields_view(t, spec, DAMPR_OP_SUM_I64);   // the table counts the lines of each key
    RecView rv{rec->rec, rec->capacity, nullptr};
    if (int r = count_records(ctx, t, tb, own_lo, own_hi, tv, rv)) return r;
    if (spec->op == DAMPR_OP_SUM_F64) return launch_fold<VK_F64, M_RECORDS>(ctx, tb, own_lo, own_hi, spec, tv, rv);
    return launch_fold<VK_INT, M_RECORDS>(ctx, tb, own_lo, own_hi, spec, tv, rv);
}

extern "C" int32_t dampr_text_json_fields(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                                          uint64_t own_hi, const dampr_fields_spec *spec,
                                          const dampr_json_members *members) {
    JsonView jv;
    JsonPathView pv;
    bool paths;
    Where w;
    if (int r = check_json_args(ctx, t, tb, own_lo, own_hi, spec, members, jv, pv, paths, w)) return r;
    const JsonPathView *p = paths ? &pv : nullptr;
    const bool f64 = spec->op == DAMPR_OP_MIN_F64 || spec->op == DAMPR_OP_MAX_F64;
    ARG_CHECK(ctx, f64 || spec->op == DAMPR_OP_SUM_I64 || spec->op == DAMPR_OP_MIN_I64 ||
                       spec->op == DAMPR_OP_MAX_I64,
              "op must be DAMPR_OP_SUM_I64, DAMPR_OP_MIN_I64, DAMPR_OP_MAX_I64, DAMPR_OP_MIN_F64 or DAMPR_OP_MAX_F64");
    ARG_CHECK(ctx, !f64 || spec->val_field != DAMPR_FIELD_VAL_ONE, "a float op needs a value field");
    if (own_hi <= own_lo) return DAMPR_OK;
    const FieldsView tv = fields_view(t, spec, spec->op);
    wait_uploads(ctx);
    if (f64) return launch_json_fold<VK_F64, M_TABLE>(ctx, tb, own_lo, own_hi, spec, jv, p, w, tv, RecView{});
    return launch_json_fold<VK_INT, M_TABLE>(ctx, tb, own_lo, own_hi, spec, jv, p, w, tv, RecView{});
}

extern "C" int32_t dampr_text_json_fields_records(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb,
                                                  uint64_t own_lo, uint64_t own_hi, const dampr_fields_spec *spec,
                                                  const dampr_json_members *members, dampr_kv *rec) {
    JsonView jv;
    JsonPathView pv;
    bool paths;
    Where w;
    if (int r = check_json_args(ctx, t, tb, own_lo, own_hi, spec, members, jv, pv, paths, w)) return r;
    const JsonPathView *p = paths ? &pv : nullptr;
    ARG_CHECK(ctx, rec != nullptr, "null");
    ARG_CHECK(ctx, spec->op == DAMPR_OP_SUM_I64 || spec->op == DAMPR_OP_SUM_F64,
              "op must be DAMPR_OP_SUM_I64 or DAMPR_OP_SUM_F64");
    ARG_CHECK(ctx, spec->val_field != DAMPR_FIELD_VAL_ONE, "record mode needs a value field");
    if (own_hi <= own_lo) return DAMPR_OK;
    const FieldsView tv = fields_view(t, spec, DAMPR_OP_SUM_I64);
    RecView rv{rec->rec, rec->capacity, nullptr};
    if (int r = count_records(ctx, t, tb, own_lo, own_hi, tv, rv)) return r;
    if (spec->op == DAMPR_OP_SUM_F64)
        return launch_json_fold<VK_F64, M_RECORDS>(ctx, tb, own_lo, own_hi, spec, jv, p, w, tv, rv);
    return launch_json_fold<VK_INT, M_RECORDS>(ctx, tb, own_lo, own_hi, spec, jv, p, w, tv, rv);
}

extern "C" int32_t dampr_text_fields_tuple(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                                           uint64_t own_hi, const dampr_fields_spec *spec,
                                           const dampr_field_keys *keys) {
    if (int r = check_fields_args(ctx, t, tb, own_lo, own_hi, spec)) return r;
    TupleView tk;
    if (int r = tuple_view(ctx, keys, tk)) return r;
    const bool f64 = spec->op == DAMPR_OP_MIN_F64 || spec->op == DAMPR_OP_MAX_F64;
    ARG_CHECK(ctx, f64 || spec->op == DAMPR_OP_SUM_I64 || spec->op == DAMPR_OP_MIN_I64 ||
                       spec->op == DAMPR_OP_MAX_I64,
              "op must be DAMPR_OP_SUM_I64, DAMPR_OP_MIN_I64, DAMPR_OP_MAX_I64, DAMPR_OP_MIN_F64 or DAMPR_OP_MAX_F64");
    ARG_CHECK(ctx, !f64 || spec->val_field != DAMPR_FIELD_VAL_ONE, "a float op needs a value field");
    if (own_hi <= own_lo) return DAMPR_OK;
    const FieldsView tv = tuple_fields_view(t, spec, spec->op, tk);
    wait_uploads(ctx);
    if (f64) return launch_fold<VK_F64, M_TABLE>(ctx, tb, own_lo, own_hi, spec, tv, RecView{}, &tk);
    return launch_fold<VK_INT, M_TABLE>(ctx, tb, own_lo, own_hi, spec, tv, RecView{}, &tk);
}

extern "C" int32_t dampr_text_fields_tuple_records(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb,
                                                   uint64_t own_lo, uint64_t own_hi, const dampr_fields_spec *spec,
                                                   const dampr_field_keys *keys, dampr_kv *rec) {
    if (int r = check_fields_args(ctx, t, tb, own_lo, own_hi, spec)) return r;
    TupleView tk;
    if (int r = tuple_view(ctx, keys, tk)) return r;
    ARG_CHECK(ctx, rec != nullptr, "null");
    ARG_CHECK(ctx, spec->op == DAMPR_OP_SUM_I64 || spec->op == DAMPR_OP_SUM_F64,
              "op must be DAMPR_OP_SUM_I64 or DAMPR_OP_SUM_F64");
    ARG_CHECK(ctx, spec->val_field != DAMPR_FIELD_VAL_ONE, "record mode needs a value field");
    if (own_hi <= own_lo) return DAMPR_OK;
    const FieldsView tv = tuple_fields_view(t, spec, DAMPR_OP_SUM_I64, tk);
    RecView rv{rec->rec, rec->capacity, nullptr};
    if (int r = count_records(ctx, t, tb, own_lo, own_hi, tv, rv)) return r;
    if (spec->op == DAMPR_OP_SUM_F64) return launch_fold<VK_F64, M_RECORDS>(ctx, tb, own_lo, own_hi, spec, tv, rv, &tk);
    return launch_fold<VK_INT, M_RECORDS>(ctx, tb, own_lo, own_hi, spec, tv, rv, &tk);
}

extern "C" int32_t dampr_table_fetch_field_keys(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, int32_t sep,
                                                const dampr_field_keys *keys, uint32_t widths[DAMPR_FIELD_KEYS_MAX],
                                                void *const cols[DAMPR_FIELD_KEYS_MAX], uint64_t *counts,
                                                uint64_t *codes, uint64_t cap, uint64_t *n) {
    ARG_CHECK(ctx, ctx && t && tb && n && widths, "null");
    ARG_CHECK(ctx, sep == DAMPR_FIELD_SEP_WS || (sep > 0 && sep < 0x80 && sep != '\n' && sep != '\r'),
              "separator must be DAMPR_FIELD_SEP_WS or an ASCII byte other than NUL, '\\n' and '\\r'");
    TupleView tk;
    if (int r = tuple_view(ctx, keys, tk)) return r;
    uint64_t st[8];
    if (int r = dampr_table_stats(ctx, t, st)) return r;
    const u64 m = *n = st[0];
    const bool ws = sep == DAMPR_FIELD_SEP_WS;
    const unsigned grid = ctx->num_sms * 4;
    if (!cols) {   // phase 1: the longest str component of each column
        for (int j = 0; j < T_MAX; ++j) widths[j] = 0;
        if (m == 0) return DAMPR_OK;
        u32 *d = (u32 *)pool_alloc(ctx, T_MAX * sizeof(u32));
        ARG_CHECK(ctx, d != nullptr, "device allocation failed");
        cudaError_t e = cudaMemsetAsync(d, 0, T_MAX * sizeof(u32), ctx->stream);
        if (e == cudaSuccess) {
            ScopedTimer tm(ctx, DAMPR_K_TABLE_EXTRACT);
            if (ws)
                table_tuple_keys_kernel<true><<<grid, 256, 0, ctx->stream>>>(
                    t->keys, t->counts, t->reps, t->cap, tb->text, (u32)sep, tk, TupleCols{}, nullptr, nullptr, 0,
                    nullptr, d);
            else
                table_tuple_keys_kernel<false><<<grid, 256, 0, ctx->stream>>>(
                    t->keys, t->counts, t->reps, t->cap, tb->text, (u32)sep, tk, TupleCols{}, nullptr, nullptr, 0,
                    nullptr, d);
            e = cudaGetLastError();
        }
        u32 w[T_MAX];
        if (e == cudaSuccess) e = cudaMemcpyAsync(w, d, sizeof w, cudaMemcpyDeviceToHost, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        pool_free(ctx, d);
        if (e != cudaSuccess) {
            ctx->err = std::string("table fetch_field_keys failed: ") + cudaGetErrorString(e);
            return DAMPR_ERR_CUDA;
        }
        for (int j = 0; j < T_MAX; ++j) widths[j] = j < tk.n && !tk.is_int[j] ? w[j] : 0;
        return DAMPR_OK;
    }
    ARG_CHECK(ctx, cap >= m, "fetch arrays too small");
    if (m == 0) return DAMPR_OK;
    // one pool block: the columns, then counts, codes and the cursor
    u64 bytes[T_MAX], total = 0;
    for (int j = 0; j < tk.n; ++j) {
        ARG_CHECK(ctx, cols[j] != nullptr, "null column");
        ARG_CHECK(ctx, tk.is_int[j] || (widths[j] >= 1 && widths[j] <= 0xFFFFFu), "a str column's width");
        bytes[j] = tk.is_int[j] ? m * 8 : ((m * widths[j] + 7) & ~7ULL);
        total += bytes[j];
    }
    u8 *d = (u8 *)pool_alloc(ctx, total + 2 * m * 8 + 8);
    ARG_CHECK(ctx, d != nullptr, "device allocation failed");
    TupleCols out{};
    u64 off = 0;
    for (int j = 0; j < tk.n; ++j) {
        if (tk.is_int[j]) out.ints[j] = (long long *)(d + off);
        else out.str[j] = d + off;
        out.width[j] = tk.is_int[j] ? 0 : widths[j];
        off += bytes[j];
    }
    u64 *d_counts = (u64 *)(d + total), *d_codes = d_counts + m, *d_cur = d_codes + m;
    cudaError_t e = cudaMemsetAsync(d_cur, 0, 8, ctx->stream);
    if (e == cudaSuccess) {
        ScopedTimer tm(ctx, DAMPR_K_TABLE_EXTRACT);
        if (ws)
            table_tuple_keys_kernel<true><<<grid, 256, 0, ctx->stream>>>(
                t->keys, t->counts, t->reps, t->cap, tb->text, (u32)sep, tk, out, d_counts, d_codes, m, d_cur,
                nullptr);
        else
            table_tuple_keys_kernel<false><<<grid, 256, 0, ctx->stream>>>(
                t->keys, t->counts, t->reps, t->cap, tb->text, (u32)sep, tk, out, d_counts, d_codes, m, d_cur,
                nullptr);
        e = cudaGetLastError();
    }
    off = 0;
    for (int j = 0; j < tk.n && e == cudaSuccess; ++j) {
        e = cudaMemcpyAsync(cols[j], d + off, tk.is_int[j] ? m * 8 : m * widths[j], cudaMemcpyDeviceToHost,
                            ctx->stream);
        off += bytes[j];
    }
    if (e == cudaSuccess && counts) e = cudaMemcpyAsync(counts, d_counts, m * 8, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess && codes) e = cudaMemcpyAsync(codes, d_codes, m * 8, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    pool_free(ctx, d);
    if (e != cudaSuccess) {
        ctx->err = std::string("table fetch_field_keys failed: ") + cudaGetErrorString(e);
        return DAMPR_ERR_CUDA;
    }
    return DAMPR_OK;
}

extern "C" int32_t dampr_text_fields_expr(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb, uint64_t own_lo,
                                          uint64_t own_hi, const dampr_fields_spec *spec, const dampr_field_expr *expr) {
    if (int r = check_fields_args(ctx, t, tb, own_lo, own_hi, spec)) return r;
    const bool f64 = spec->op == DAMPR_OP_MIN_F64 || spec->op == DAMPR_OP_MAX_F64;
    ARG_CHECK(ctx, f64 || spec->op == DAMPR_OP_SUM_I64 || spec->op == DAMPR_OP_MIN_I64 ||
                       spec->op == DAMPR_OP_MAX_I64,
              "op must be DAMPR_OP_SUM_I64, DAMPR_OP_MIN_I64, DAMPR_OP_MAX_I64, DAMPR_OP_MIN_F64 or DAMPR_OP_MAX_F64");
    TupleView tk;
    ExprView xe;
    if (int r = expr_view(ctx, expr, f64, tk, xe)) return r;
    ARG_CHECK(ctx, !f64 || xe.val_len || spec->val_field != DAMPR_FIELD_VAL_ONE, "a float op needs a value");
    if (own_hi <= own_lo) return DAMPR_OK;
    const FieldsView tv = fields_view(t, spec, spec->op);
    wait_uploads(ctx);
    if (f64) return launch_fold<VK_F64, M_TABLE>(ctx, tb, own_lo, own_hi, spec, tv, RecView{}, &tk, &xe);
    return launch_fold<VK_INT, M_TABLE>(ctx, tb, own_lo, own_hi, spec, tv, RecView{}, &tk, &xe);
}

extern "C" int32_t dampr_text_fields_expr_records(dampr_ctx *ctx, dampr_table *t, dampr_textbuf *tb,
                                                  uint64_t own_lo, uint64_t own_hi, const dampr_fields_spec *spec,
                                                  const dampr_field_expr *expr, dampr_kv *rec) {
    if (int r = check_fields_args(ctx, t, tb, own_lo, own_hi, spec)) return r;
    ARG_CHECK(ctx, rec != nullptr, "null");
    ARG_CHECK(ctx, spec->op == DAMPR_OP_SUM_I64 || spec->op == DAMPR_OP_SUM_F64,
              "op must be DAMPR_OP_SUM_I64 or DAMPR_OP_SUM_F64");
    TupleView tk;
    ExprView xe;
    if (int r = expr_view(ctx, expr, spec->op == DAMPR_OP_SUM_F64, tk, xe)) return r;
    ARG_CHECK(ctx, xe.val_len || spec->val_field != DAMPR_FIELD_VAL_ONE, "record mode needs a value");
    if (own_hi <= own_lo) return DAMPR_OK;
    const FieldsView tv = fields_view(t, spec, DAMPR_OP_SUM_I64);   // the table counts the lines of each key
    RecView rv{rec->rec, rec->capacity, nullptr};
    if (int r = count_records(ctx, t, tb, own_lo, own_hi, tv, rv)) return r;
    if (spec->op == DAMPR_OP_SUM_F64)
        return launch_fold<VK_F64, M_RECORDS>(ctx, tb, own_lo, own_hi, spec, tv, rv, &tk, &xe);
    return launch_fold<VK_INT, M_RECORDS>(ctx, tb, own_lo, own_hi, spec, tv, rv, &tk, &xe);
}
