"""The numpy stand-in of tests/fields_standin.py with the WHERE predicates of dampr_text_fields and
dampr_text_fields_records (include/dampr_b200.h): the tests of `filter(...)` in front of a field fold
(test_text_fields_where_lowering.py) run on it. Without predicates a table behaves exactly like the plain stand-in's.

Per line the device can take (ASCII, no NUL, no text-mode '\\r', under 4 KB), the predicates are evaluated in order:
the first false one drops the line (a hole in record mode, stats[6] in table mode), the first one the device cannot
decide hands the line back as a fallback line, and a line that passes all of them is the plain stand-in's."""
from fields_standin import _int18, device_takes, make_ctx, parse_f64

_CMPS = [lambda x, c: x == c, lambda x, c: x != c, lambda x, c: x < c, lambda x, c: x <= c, lambda x, c: x > c,
         lambda x, c: x >= c]


def where(f, preds):
    """the header's WHERE rule over the split line f (bytes fields): True if every predicate holds, False at the
    first false one, None at the first one the device cannot decide (the host's Python then decides)"""
    from dampr_b200 import device as dev
    for kind, i, cmp, consts in preds:
        if kind == dev.PRED_NFIELDS:
            x = len(f)
        elif not -len(f) <= i < len(f):
            return None
        elif kind == dev.PRED_STR:
            x, consts = f[i], [c.encode("utf-8") for c in consts]
        else:
            x = _int18(f[i]) if kind == dev.PRED_INT else parse_f64(f[i])
            if x is None:
                return None
        if cmp in (dev.CMP_IN, dev.CMP_NOT_IN):
            r = (x in consts) == (cmp == dev.CMP_IN)
        else:
            r = _CMPS[cmp](x, consts[0])
        if not r:
            return False
    return True


def line_verdict(line, f, preds, cr_is_data):
    """the WHERE rule of one line whose fields are f: False (dropped), None (the host's: a line the device does not
    take, or a predicate it cannot decide) or True (the key and value decide)"""
    if not device_takes(line, cr_is_data):
        return None
    return where(f, preds) if preds else True


def make_where_ctx(free_bytes=1 << 30):
    """make_ctx(free_bytes) whose tables also take the `preds` of fields() and fields_records()"""
    from dampr_b200 import device as dev
    ctx = make_ctx(free_bytes)
    Base = type(ctx.table(4))

    class WhereTable(Base):
        _preds = ()

        def fields(self, tb, lo, hi, spec, cr_is_data=False, preds=()):
            dev.fields_spec(spec, cr_is_data, preds)   # the binding's packing of the predicates
            self._preds = tuple(preds)
            Base.fields(self, tb, lo, hi, spec, cr_is_data)

        def fields_records(self, tb, lo, hi, spec, kv, cr_is_data=False, preds=()):
            dev.fields_spec(spec, cr_is_data, preds)
            self._preds = tuple(preds)
            Base.fields_records(self, tb, lo, hi, spec, kv, cr_is_data)

        def _line(self, line, off, sep, kf, kind, vf, op, cr_is_data, rec):
            verdict = line_verdict(line, line.split(sep), self._preds, cr_is_data)
            if verdict is False:      # dropped: a hole in record mode, counted in stats[6] in table mode
                if rec is not None:
                    self._put(rec, 0, 0)
                else:
                    self.st["raw"] += 1
            elif verdict is None:     # the host's filters decide
                self._hand_back(line, off, rec)
            else:
                Base._line(self, line, off, sep, kf, kind, vf, op, cr_is_data, rec)

        def _hand_back(self, line, off, rec):
            st = self.st
            if len(line) > 0xFFFF:
                st["flags"] |= dev.TF_LONGLINE
            elif len(self.fb) < (1 << 16):
                self.fb.append((off << 16) | len(line))
                st["fallback"] += 1
            else:
                st["flags"] |= dev.TF_NONASCII
            if rec is not None:
                self._put(rec, 0, 0)

    ctx.table = lambda log2: WhereTable(ctx, log2)
    return ctx
