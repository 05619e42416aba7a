"""The numpy stand-in of tests/fields_where_standin.py with the whitespace split of dampr_text_fields and
dampr_text_fields_records (sep == DAMPR_FIELD_SEP_WS, include/dampr_b200.h): the tests of `line.split()` field folds
(test_text_fields_ws_lowering.py) run on it. With a separator byte a table behaves exactly like the WHERE stand-in's.

Under DAMPR_FIELD_SEP_WS a line's fields are str.split() of the decoded line, never bytes.split(): the two differ on
0x1C-0x1F, which str.split() takes as whitespace. The plain and WHERE stand-ins read the fields through
`line.split(sep)`, so the line is handed to them as a bytes object whose split() is str.split()."""
from fields_where_standin import make_where_ctx


class WsLine(bytes):
    """a line whose split() is str.split() of the decoded line (the device's lines are ASCII; others go to the host
    whatever their fields)"""
    def split(self, sep=None, maxsplit=-1):
        return [f.encode("utf-8", "surrogateescape")
                for f in self.decode("utf-8", "surrogateescape").split()]


def ws_field_offsets(line):
    """byte offset in `line` (ASCII bytes) of each of its str.split() fields"""
    out, pos = [], 0
    for f in WsLine(line).split():
        pos = line.index(f, pos)
        out.append(pos)
        pos += len(f)
    return out


def make_ws_ctx(free_bytes=1 << 30):
    """make_where_ctx(free_bytes) whose tables also take sep == FIELD_SEP_WS"""
    from dampr_b200 import device as dev
    ctx = make_where_ctx(free_bytes)
    Base = type(ctx.table(4))

    class WsTable(Base):
        def _scan(self, tb, lo, hi, spec, cr_is_data, rec):
            if spec[0] != dev.FIELD_SEP_WS:
                return Base._scan(self, tb, lo, hi, spec, cr_is_data, rec)
            _sep, kf, kind, vf, op = spec
            data = tb.buf[:tb.n].tobytes()
            pos = 0
            while pos < len(data):
                end = data.find(b"\n", pos)
                end = len(data) if end < 0 else end
                if lo <= pos < hi:
                    self._ws_line(WsLine(data[pos:end]), pos, kf, kind, vf, op, cr_is_data, rec)
                pos = end + 1

        def _ws_line(self, line, off, kf, kind, vf, op, cr_is_data, rec):
            key, folded = None, self.st["folded"]
            if kind == dev.FIELD_KEY_STR:
                f = line.split()
                if -len(f) <= kf < len(f) and not 1 <= len(f[kf]) <= 9:
                    key, old = f[kf], self.rep.get(f[kf])
            # the WHERE stand-in's rules with the fields of str.split(); the representative of a hashed key is
            # restated with the key's real offset (the plain stand-in adds one byte per separator)
            Base._line(self, line, off, None, kf, kind, vf, op, cr_is_data, rec)
            if key is not None and self.st["folded"] > folded:
                k_off = off + ws_field_offsets(line)[kf]
                self.rep[key] = min(old if old is not None else 1 << 62, (k_off << 20) | len(key))

    ctx.table = lambda log2: WsTable(ctx, log2)
    return ctx
