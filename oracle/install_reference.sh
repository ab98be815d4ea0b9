#!/bin/bash
# Offline install of the UNMODIFIED reference package (baybe) into oracle/_ref (git-ignored), for the tests that
# drive the plugin through the reference's own Campaign.  The source tree is read-only and its pyproject lists only the top-level package (the sub-packages are picked up
# by setuptools_scm's file finder, which is not installed here), so the install runs from a /tmp copy whose
# packaging table -- nothing else -- is switched to `packages.find`.  Dependencies are not resolvable offline
# (--no-deps): botorch / gpytorch / cattrs are absent, so only the parts of baybe that do not import them run
# (Campaign, search spaces, the recommender base classes); tests/shims/cattrs stands in for cattrs.
set -e
cd "$(dirname "$0")/.."
SRC=${1:-/root/reference}
[ -d "$SRC/baybe" ] || { echo "no reference tree at $SRC"; exit 0; }
if [ -f oracle/_ref/baybe/recommenders/pure/bayesian/base.py ]; then echo "oracle/_ref present"; exit 0; fi
TMP=$(mktemp -d)
cp -r "$SRC" "$TMP/ref"
python - "$TMP/ref/pyproject.toml" <<'PY'
import sys
p = sys.argv[1]
s = open(p).read()
s = s.replace('[tool.setuptools]\npackages = ["baybe"]', '[tool.setuptools.packages.find]\ninclude = ["baybe*"]')
open(p, "w").write(s)
PY
rm -rf oracle/_ref
python -m pip install -q --no-index --no-build-isolation --no-deps --target oracle/_ref "$TMP/ref"
rm -rf "$TMP"
echo "installed $(find oracle/_ref/baybe -name '*.py' | wc -l) modules into oracle/_ref"
