"""One pass of each kv hot kernel on device-resident synthetic records, for ncu captures:
    ncu --set full --import-source on --clock-control none \
        -k regex:"part_hist2|part_scatter|leaf_sort|merge_tile" -c 8 -o kv_one python tools/kv_one.py 40"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dampr_b200 import device as dev


def main():
    n = int(float(sys.argv[1]) * 1e6) if len(sys.argv) > 1 else 40_000_000
    ctx = dev.Ctx(0)
    kv = ctx.synth_kv(42, n, n)
    kv.sort(dev.KEY_MIX)
    ctx.sync()
    red = kv.reduce_by_key(dev.OP_SUM_I64)
    ctx.sync()
    red.free()
    kv.free()
    runs = []
    for s in range(8):
        r = ctx.synth_kv(100 + s, n // 8, n)
        r.sort(dev.KEY_MIX)
        runs.append(r)
    ctx.sync()
    m = ctx.kv_merge(runs, dev.KEY_MIX, -1)
    ctx.sync()
    print("sorted %d, merged %d" % (n, len(m)))
    ctx.close()


if __name__ == "__main__":
    main()
