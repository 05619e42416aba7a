"""Ad-hoc device timings (development aid): python tools/quick_bench.py [text_gb] [kv_mrec]"""
import ctypes as C
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dampr_b200 import device as dev
from oracle import gen


def synth_text(ctx, n_lines, V, seed=1234):
    vocab = gen.make_vocab(V)
    cdf = gen.make_cdf(V)
    cap = int(n_lines * 110) + (1 << 20)
    tb = ctx.textbuf(cap)
    out = C.c_uint64(0)
    vb, vo = vocab
    ctx.check(ctx.lib.dampr_synth_text(ctx.h, tb.h, seed, n_lines, vb.ctypes.data_as(C.c_void_p),
                                       vo.ctypes.data_as(C.c_void_p), V, cdf.ctypes.data_as(C.c_void_p),
                                       C.byref(out)))
    tb.n = out.value
    return tb


def summarize(ctx, label, nbytes):
    tms = ctx.timings()
    agg = {}
    for name, ms in tms:
        agg.setdefault(name, [0, 0.0])
        agg[name][0] += 1
        agg[name][1] += ms
    tot = sum(v[1] for v in agg.values())
    print("%s: total %.3f ms  -> %.1f GB/s" % (label, tot, nbytes / tot / 1e6 if tot else 0))
    for k, (c, ms) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("    %-14s x%-4d %9.3f ms" % (k, c, ms))
    ctx.timings_reset()


def main():
    text_gb = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    kv_mrec = float(sys.argv[2]) if len(sys.argv) > 2 else 100.0
    ctx = dev.Ctx(0)
    if text_gb > 0:
        n_lines = int(text_gb * 1e9 / 99.0)
        t0 = time.time()
        tb = synth_text(ctx, n_lines, 1000000)
        ctx.sync()
        print("synth text: %d bytes, %d lines in %.2fs" % (tb.n, n_lines, time.time() - t0))
        ctx.timings_reset()
        for mode, name, ctas in ((dev.TOK_NONWORD_LOWER_SET, "tfidf-set-3cta", 3), (dev.TOK_NONWORD_LOWER_SET, "tfidf-set-4cta", 4),
                                 (dev.TOK_NONWORD_LOWER_SET, "tfidf-set-2cta", 2),
                                 (dev.TOK_WS, "wc-split-3cta", 3), (dev.TOK_WS, "wc-split-4cta", 4),
                                 (dev.TOK_NONWORD_LOWER, "nonword-3cta", 3), (dev.TOK_NONWORD_LOWER, "nonword-4cta", 4)):
            if os.environ.get("QB_ONLY") and os.environ["QB_ONLY"] != name:
                continue
            dev.set_option("text_ctas", ctas)
            for rep in range(3):
                tab = ctx.table(21)
                ctx.sync()
                ctx.timings_reset()
                tab.count(tb, 0, tb.n, mode)
                st = tab.stats()
                summarize(ctx, "text_count[%s] rep%d entries=%d lines=%d hashed=%d flags=%d" % (
                    name, rep, st["entries"], st["lines"], st["hashed"], st["flags"]), tb.n)
                if rep == 2 and st["hashed"]:
                    tab.verify(tb, 0, tb.n, mode)
                    st2 = tab.stats()
                    summarize(ctx, "text_verify[%s] flags=%d" % (name, st2["flags"]), tb.n)
                tab.free()
        tb.free()
    if kv_mrec > 0:
        n = int(kv_mrec * 1e6)
        for nk, label in ((10_000_000, "K=1e7"), (n, "K=N")):
            kv = ctx.kv(n)
            ctx.check(ctx.lib.dampr_synth_kv(ctx.h, kv.h, 42, n, nk))
            ctx.sync()
            ctx.timings_reset()
            t0 = time.time()
            kv.sort(dev.KEY_MIX)
            ctx.sync()
            wall = time.time() - t0
            summarize(ctx, "kv_sort[%s] n=%d wall=%.1fms" % (label, n, wall * 1e3), 32 * n)
            ctx.check(ctx.lib.dampr_synth_kv(ctx.h, kv.h, 42, n, nk))
            ctx.sync()
            ctx.timings_reset()
            t0 = time.time()
            out = kv.sort_reduce(dev.OP_SUM_I64, dev.KEY_MIX)
            ctx.sync()
            wall = time.time() - t0
            summarize(ctx, "kv_sort_reduce[%s] n=%d groups=%d wall=%.1fms" % (label, n, len(out), wall * 1e3),
                      16 * n + 16 * len(out))
            out.free()
            kv.free()
    ctx.close()


if __name__ == "__main__":
    main()
