#!/bin/sh
# Installs the UNMODIFIED reference (Refefer/Dampr, pure Python) from a checkout of it (argument 1) into
# oracle/_ref/ with pip. oracle/_ref/ is git-ignored (no reference source enters the history); where it is present,
# bench.py --impl reference and the bench's parity check run the real reference on the host cores.
# The checkout may be read-only and setup.py writes build/ + egg-info next to itself: install from a copy.
# The reference's own test package is left out: pytest would collect it from the tree.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
SRC="${1:-/root/reference}"
[ -d "$SRC/dampr" ] || { echo "no reference checkout at $SRC" >&2; exit 3; }
TMP="$(mktemp -d /tmp/dampr_ref_src.XXXXXX)"
cp -r "$SRC/." "$TMP/"
rm -rf "$HERE/_ref"
mkdir -p "$HERE/_ref"
python -m pip install --quiet --no-index --no-build-isolation --no-deps --find-links /opt/wheelhouse \
    --target "$HERE/_ref" "$TMP"
rm -rf "$TMP" "$HERE/_ref/tests"
python - "$HERE/_ref" <<'PY'
import sys
sys.path.insert(0, sys.argv[1])
import dampr
assert dampr.__file__.startswith(sys.argv[1]), dampr.__file__
print("reference installed:", dampr.__file__)
PY
