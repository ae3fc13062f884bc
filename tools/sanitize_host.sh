#!/bin/sh
# ThreadSanitizer and Address/UB-Sanitizer runs of the CPU side of libb200kv (pool, hash, cache server
# and client, disk tier) under a multi-threaded stress driver.  Usage: tools/sanitize_host.sh [iterations]
set -e
here="$(cd "$(dirname "$0")/.." && pwd)"
src="$here/production-stack_b200/csrc"
out="${TMPDIR:-/tmp}/b200kv-sanitize"
mkdir -p "$out"
for san in thread address,undefined; do
  name=$(echo "$san" | tr ',' '_')
  g++ -std=c++17 -O1 -g -fsanitize=$san -fno-omit-frame-pointer -I"$here/include" \
      "$src/b200kv_pool.cpp" "$src/b200kv_hash.cpp" "$src/b200kv_remote.cpp" "$src/b200kv_disk.cpp" "$here/tools/sanitize_host.cpp" \
      -o "$out/stress_$name" -lpthread -lrt
  echo "== -fsanitize=$san"
  "$out/stress_$name" "${1:-20000}"
done
