#!/bin/bash
# Build the reference arm of bench.py (`--impl reference`, `gpu_eager_baseline`): a copy of the unmodified original
# project's `core` package in oracle/_ref/core (git-ignored).  The original is pure Python, so building it is copying it.
# Source: $RNC_REFERENCE, or a checkout named `reference` beside this repository.  Without one, nothing is built and
# bench.py times the oracle port instead.
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF=${RNC_REFERENCE:-$(dirname "$(dirname "$HERE")")/reference}
[ -d "$REF/core" ] || { echo "no original project at $REF: reference arm not built"; exit 0; }
rm -rf "$HERE/_ref"
mkdir -p "$HERE/_ref"
cp -r "$REF/core" "$HERE/_ref/core"
echo "reference arm: $HERE/_ref/core"
