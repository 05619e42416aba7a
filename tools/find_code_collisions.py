"""Find pairs of different long tokens that share a 64-bit key code, for tests/golden/code_collisions.json.

Tokens too long for an exact code (csrc/text2.cu token_code2, csrc/text.cu token_code, csrc/fields.cu hash_bytes) get
    1 << 63 | mix64((h1 << 32 | h2) ^ len * 0x9E3779B97F4A7C15)
where h1 and h2 are two 32-bit running hashes under the fixed seed 0x243F6A8885A308D3, fed with the bytes as they are
(`raw`: str.split tokens and field keys) or with the [^\\w]+ symbols 0-9 -> 1..10, '_' -> 11, letters case-folded to
12..37 (`sym`). Both updates are bijections of the state, so a parallel Pollard-rho search with distinguished points
finds two 13-character tokens with equal (h1, h2) states in seconds. A state-level pair collides after any common
suffix too; a pair that only agrees after mix64 and bit 63 would not, and this search never yields one.

Tokens are 13 characters of the 32-letter alphabet below (word characters only, no separators): character i is
ALPHABET[(x >> 5i) & 31] of a 64-bit x, so distinct x give distinct tokens. The rho function maps x to the state of
its token. Trails start from splitmix64(seed, index), run in batches in parallel and are merged in index order, so
the output depends on the seed alone, not on the number of threads.

    python tools/find_code_collisions.py [--seed 1] [--pairs 4] [--out tests/golden/code_collisions.json]

Needs gcc with OpenMP; about two minutes on 8 cores for the default four pairs of each variant.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

SEED = 0x243F6A8885A308D3
ALPHABET = "abcdefghijklmnopqrstuvwxyz012345"
LENGTH = 13
M64 = (1 << 64) - 1
M32 = (1 << 32) - 1

C_SRC = r"""
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
typedef uint64_t u64;
typedef uint32_t u32;

static u32 VT[32];                 /* hash input of each alphabet letter */
static const char *ALPHA = "%(alphabet)s";

static inline u64 f(u64 x) {
    u32 h1 = (u32)%(seed)dULL ^ 0x811C9DC5u, h2 = (u32)(%(seed)dULL >> 32) ^ 0x9747B28Cu;
    for (int i = 0; i < %(length)d; ++i) {
        const u32 v = VT[(x >> (5 * i)) & 31];
        h1 = (h1 ^ v) * 16777619u;
        h2 = (h2 ^ v) * 0x85EBCA6Bu + 0x9E3779B9u;
        h2 = (h2 << 13) | (h2 >> 19);
    }
    return ((u64)h1 << 32) | h2;
}

static u64 splitmix(u64 z) {
    z += 0x9E3779B97F4A7C15ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}

static void put_token(u64 x) {
    char t[%(length)d + 1];
    for (int i = 0; i < %(length)d; ++i) t[i] = ALPHA[(x >> (5 * i)) & 31];
    t[%(length)d] = 0;
    fputs(t, stdout);
}

#define DP_BITS 14
#define MAX_TRAIL (40u << DP_BITS)
#define BATCH 4096
#define MAP_LOG 22
typedef struct { u64 dp, start; u32 len, used; } Entry;

int main(int argc, char **argv) {
    const int sym = atoi(argv[1]);
    const u64 seed = strtoull(argv[2], 0, 0);
    const int want = atoi(argv[3]);
    for (int i = 0; i < 32; ++i) {
        const u32 c = (unsigned char)ALPHA[i];
        VT[i] = !sym ? c : (c >= '0' && c <= '9') ? c - '0' + 1 : c == '_' ? 11 : (c | 0x20) - 'a' + 12;
    }
    Entry *map = calloc((size_t)1 << MAP_LOG, sizeof(Entry));
    u64 found[64];
    int nfound = 0;
    u64 starts[BATCH], dps[BATCH];
    u32 lens[BATCH];
    for (u64 batch = 0; nfound < want; ++batch) {
        #pragma omp parallel for schedule(dynamic, 16)
        for (int i = 0; i < BATCH; ++i) {
            const u64 s = splitmix(seed * 0x100000001B3ULL ^ splitmix(batch * BATCH + i));
            u64 x = s;
            u32 n = 0;
            while ((x & ((1u << DP_BITS) - 1)) != 0 && n < MAX_TRAIL) {
                x = f(x);
                ++n;
            }
            starts[i] = s;
            dps[i] = x;
            lens[i] = (x & ((1u << DP_BITS) - 1)) == 0 ? n : 0;   /* 0: no distinguished point (a cycle) */
        }
        for (int i = 0; i < BATCH && nfound < want; ++i) {
            if (!lens[i]) continue;
            u64 h = splitmix(dps[i]) >> (64 - MAP_LOG);
            while (map[h].used && map[h].dp != dps[i]) h = (h + 1) & (((u64)1 << MAP_LOG) - 1);
            if (!map[h].used) {
                map[h] = (Entry){dps[i], starts[i], lens[i], 1};
                continue;
            }
            /* two trails meet at one distinguished point: walk them to where they merge */
            u64 a = map[h].start, b = starts[i];
            u32 la = map[h].len, lb = lens[i];
            for (; la > lb; --la) a = f(a);
            for (; lb > la; --lb) b = f(b);
            u64 fa = f(a), fb = f(b);
            while (a != b && fa != fb) {
                a = fa;
                b = fb;
                fa = f(a);
                fb = f(b);
            }
            if (a == b) continue;   /* one trail started on the other */
            int dup = 0;
            for (int k = 0; k < nfound; ++k) dup |= found[k] == fa;
            if (dup) continue;
            found[nfound++] = fa;
            if (a > b) { u64 t = a; a = b; b = t; }
            put_token(a);
            putchar(' ');
            put_token(b);
            printf(" %%016llx\n", (unsigned long long)fa);
            fflush(stdout);
        }
    }
    free(map);
    return 0;
}
"""


def mix64(x):
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & M64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def state(token, variant):
    """(h1 << 32 | h2) after the bytes of token (the kernels' running hashes)"""
    h1, h2 = (SEED & M32) ^ 0x811C9DC5, (SEED >> 32) ^ 0x9747B28C
    for c in token.encode("ascii"):
        if variant == "sym":
            c = c - 0x2F if 0x30 <= c <= 0x39 else (11 if c == 0x5F else ((c & 0x7F) | 0x20) - 0x55)
        h1 = ((h1 ^ c) * 16777619) & M32
        h2 = ((h2 ^ c) * 0x85EBCA6B + 0x9E3779B9) & M32
        h2 = ((h2 << 13) | (h2 >> 19)) & M32
    return (h1 << 32) | h2


def code(token, variant):
    return mix64(state(token, variant) ^ ((len(token) * 0x9E3779B97F4A7C15) & M64)) | (1 << 63)


def search(variant, seed, pairs, workdir):
    src = os.path.join(workdir, "rho.c")
    exe = os.path.join(workdir, "rho")
    with open(src, "w") as f:
        f.write(C_SRC % {"alphabet": ALPHABET, "seed": SEED, "length": LENGTH})
    subprocess.check_call(["gcc", "-O3", "-fopenmp", "-o", exe, src])
    out = subprocess.check_output([exe, "1" if variant == "sym" else "0", str(seed), str(pairs)]).decode()
    found = []
    for line in out.splitlines():
        a, b, st = line.split()
        assert a != b and state(a, variant) == state(b, variant) == int(st, 16), line
        found.append({"a": a, "b": b, "state": "0x%016x" % state(a, variant), "code": "0x%016x" % code(a, variant)})
    return found


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--pairs", type=int, default=4, help="pairs per variant")
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                 "tests", "golden", "code_collisions.json"))
    args = ap.parse_args()
    doc = {"seed": args.seed, "hash_seed": "0x%016x" % SEED, "length": LENGTH, "alphabet": ALPHABET, "variants": {}}
    with tempfile.TemporaryDirectory() as d:
        for variant in ("raw", "sym"):
            doc["variants"][variant] = search(variant, args.seed, args.pairs, d)
            print(variant, doc["variants"][variant], file=sys.stderr)
    with open(args.out, "w") as f:
        json.dump(doc, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
