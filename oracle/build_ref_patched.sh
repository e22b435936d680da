#!/bin/bash
# Builds the reference WITH baseline/patches/*.patch applied (the multi-tile plugin seam, SURVEY.md 8b) into
# oracle/_ref/grok_patched/bin/.  The patch is applied to a scratch copy of the reference tree under oracle/_ref/_build/;
# the reference tree itself is never written.  The unmodified build (oracle/build_ref.sh -> oracle/_ref/grok) stays the
# reference arm; this one is only the host that exercises the patched per-tile binding in tests.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
SRC="${GROK_SRC:-/root/reference}"
[ -d "$SRC/src/lib/core" ] || { echo "no reference tree at $SRC"; exit 0; }
COPY="$HERE/_ref/_build/patched_src"
PATCHES="$HERE/../baseline/patches"
if [ ! -f "$COPY/.patched" ] || [ "$PATCHES/0001-multi-tile-plugin-encode-decode.patch" -nt "$COPY/.patched" ]; then
  rm -rf "$COPY"; mkdir -p "$HERE/_ref/_build"
  cp -r "$SRC" "$COPY"; rm -rf "$COPY/.git"
  for p in "$PATCHES"/*.patch; do patch -s -p1 -d "$COPY" < "$p"; done
  touch "$COPY/.patched"
fi
GROK_SRC="$COPY" GROK_BUILD_DIR="$HERE/_ref/_build/patched" GROK_OUT_DIR="$HERE/_ref/grok_patched" bash "$HERE/build_ref.sh"
