#!/bin/sh
# Builds the reference's UNMODIFIED KITTI scorer (src/dataset/kitti-eval/cpp/evaluate_object.cpp,
# recipe = its own one-line Makefile: `g++ -Wall -Wno-sign-compare`) from the sources where they
# lie in the reference checkout, into oracle/_ref/evaluate_object - the path
# squeezedet_b200/eval.py shells out to, mirroring src/dataset/kitti.py:129-136.
# No reference source is copied into this repo; oracle/_ref/ is git-ignored.
# Usage: oracle/build_kitti_eval.sh /path/to/reference
set -e
REF="$1"
SRC="$REF/src/dataset/kitti-eval/cpp/evaluate_object.cpp"
HERE="$(cd "$(dirname "$0")/.." && pwd)"
OUT="$HERE/oracle/_ref"
if [ ! -f "$SRC" ]; then
  echo "build_kitti_eval: $SRC not found (pass the reference checkout as the first argument)" >&2
  exit 2
fi
mkdir -p "$OUT"
g++ -O2 -Wall -Wno-sign-compare -Wno-unused-variable -Wno-unused-result \
    -I "$REF/src/dataset/kitti-eval/cpp" -o "$OUT/evaluate_object" "$SRC"
echo "built $OUT/evaluate_object"
