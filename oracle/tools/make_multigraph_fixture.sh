#!/bin/bash
# TEST INFRASTRUCTURE.  Regenerates tests/golden/multigraph_euler: the JSON of make_multigraph_json.py converted by the
# reference's OWN converter, exactly as make_tiny_fixture.sh converts the reference's test graph (scratch copy of the tools,
# three-argument form: no index step).  Only runs where /root/reference exists.  Output dir: ${1:-tests/golden/multigraph_euler}
set -euo pipefail
HERE=$(cd "$(dirname "$0")" && pwd)
OUT=${1:-$HERE/../../tests/golden/multigraph_euler}
JSON=$(mktemp /tmp/multigraph.XXXXXX.json)
python "$HERE/make_multigraph_json.py" "$JSON"
REF=${REF:-/root/reference}
PKG=$(mktemp -d /tmp/euler_tools_pkg.XXXXXX)
mkdir -p "$PKG/euler"
cp -r "$REF/euler/tools" "$PKG/euler/tools"
: > "$PKG/euler/__init__.py"
CXX="g++ -std=c++11 -O2 -fPIC -include cstdint -D_GLIBCXX_USE_CXX11_ABI=0 -I$REF"
$CXX -shared -o "$PKG/euler/tools/libcommon.so" "$REF/euler/common/hash.cc"
$CXX -shared -o "$PKG/euler/tools/libeuler_util.so" "$REF/euler/util/python_api.cc" "$REF/euler/common/hash.cc"
rm -rf "$OUT"; mkdir -p "$OUT"
PYTHONPATH="$PKG" python "$PKG/euler/tools/generate_euler_data.py" "$JSON" "$OUT" 2 >/dev/null
rm -rf "$PKG" "$JSON"
find "$OUT" -type f | sort
