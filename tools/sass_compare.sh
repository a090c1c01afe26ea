#!/bin/sh
# tools/sass_compare.sh OLD.so NEW.so
# Every kernel instance of OLD.so must exist in NEW.so with byte-identical SASS (instruction addresses aside);
# kernels only NEW.so has are listed.  Used to show that a change adds kernels without touching existing ones:
#   git stash && python -c "import __graft_entry__ as g; g.build()" && cp vorbis_b200/libvorbis_b200.so /tmp/old.so
#   git stash pop && python -c "import __graft_entry__ as g; g.build()"
#   tools/sass_compare.sh /tmp/old.so vorbis_b200/libvorbis_b200.so
set -e
CUOBJDUMP=${CUOBJDUMP:-/usr/local/cuda/bin/cuobjdump}
d=$(mktemp -d)
trap 'rm -rf "$d"' EXIT
split() {
  mkdir -p "$2"
  "$CUOBJDUMP" -sass "$1" | awk -v out="$2" '
    /Function : / { f = $3; next }
    f != "" { sub(/\/\*[0-9a-f]+\*\/ */, ""); print > (out "/" f ".sass") }'
}
split "$1" "$d/old"
split "$2" "$d/new"
n=0; bad=0
for f in "$d"/old/*.sass; do
  k=$(basename "$f" .sass); n=$((n + 1))
  if [ ! -f "$d/new/$k.sass" ]; then echo "MISSING: $k"; bad=$((bad + 1))
  elif ! cmp -s "$f" "$d/new/$k.sass"; then echo "DIFFERENT: $k"; bad=$((bad + 1)); fi
done
for f in "$d"/new/*.sass; do
  k=$(basename "$f" .sass)
  [ -f "$d/old/$k.sass" ] || echo "new: $k"
done
echo "$n kernels of $1 compared: $bad differ or are missing"
[ "$bad" -eq 0 ]
