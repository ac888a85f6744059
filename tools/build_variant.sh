#!/usr/bin/env bash
# Builds the library with extra compile flags into its own directory, leaving the in-tree build alone:
#   bash tools/build_variant.sh OUT_DIR [-DFLAG ...]   ->  OUT_DIR/libnphm_b200.so (objects and ptxas logs in OUT_DIR/obj)
# Load it with NPHM_B200_LIB=OUT_DIR/libnphm_b200.so, e.g. the timeline builds -DNPHM_ENS_TRACE (tools/ens_trace.py) and
# -DNPHM_TCL_TRACE (tools/tcl_trace.py).
set -euo pipefail
if [ $# -lt 1 ]; then
    echo "usage: $0 OUT_DIR [-DFLAG ...]" >&2
    exit 2
fi
out=$(mkdir -p "$1" && cd "$1" && pwd)
shift
here=$(cd "$(dirname "$0")/.." && pwd)
make -C "$here/nphm_b200/csrc" -j8 BUILD="$out/obj" TARGET="$out/libnphm_b200.so" EXTRA="$*"
