#!/usr/bin/env bash
# Runs tests/test_emu_kernels.py (the SIMT kernels compiled for the host, tests/emu) under
# ThreadSanitizer — a missing __syncthreads() shows up as a data race on the emulated shared
# memory — and AddressSanitizer — out-of-bounds global / shared accesses.  CPU only.
#   scripts/emu_sanitize.sh [thread|address ...] [tests/test_emu_<x>.py ...]
#   (default: both sanitizers, tests/test_emu_kernels.py)   report -> stdout
set -u
cd "$(dirname "$0")/.."
CXX=/usr/bin/g++
sans=()
tests=()
for a in "$@"; do
  case $a in
    *.py|*::*) tests+=("$a") ;;
    *) sans+=("$a") ;;
  esac
done
[ ${#sans[@]} -eq 0 ] && sans=("thread address")
[ ${#tests[@]} -eq 0 ] && tests=(tests/test_emu_kernels.py)
for san in "${sans[@]}"; do
  for s in $san; do
    lib=$(python -c "from tests import emu; print(emu.build(sanitize='$s'))") || exit 1
    case $s in
      thread)  rt=$($CXX -print-file-name=libtsan.so); opts="TSAN_OPTIONS=halt_on_error=0:report_signal_unsafe=0" ;;
      address) rt=$($CXX -print-file-name=libasan.so); opts="ASAN_OPTIONS=detect_leaks=0" ;;
      *) echo "unknown sanitizer $s"; exit 2 ;;
    esac
    echo "== $s sanitizer: $lib"
    log=$(mktemp)
    env LD_PRELOAD="$rt" $opts SRCV_EMU_LIB="$lib" python -m pytest "${tests[@]}" -q -x -s -p no:cacheprovider >"$log" 2>&1
    rc=$?
    tail -n 3 "$log"
    echo "pytest exit code: $rc"
    # reports are counted only if a frame is in our code (libtorch's own OpenMP pool trips TSan too)
    python - "$log" <<'PY'
import re, sys
txt = open(sys.argv[1], errors="replace").read()
reps = re.split(r"(?=WARNING: ThreadSanitizer|ERROR: AddressSanitizer)", txt)[1:]
# only the two ACCESS stacks count (not where the threads were created); an access inside our
# kernels / launchers has a csrc frame
def access_stacks(r):
    return re.split(r"\n\s+(?:Location is|Thread T\d+ )", r)[0]
# ... and reports with libtorch / libgomp on one side are their worker pool re-using a main-thread
# stack slot (libgomp's synchronisation is invisible to TSan)
ours = [r for r in reps if "simplerecon_b200/csrc" in access_stacks(r)
        and "libtorch" not in access_stacks(r) and "libgomp" not in access_stacks(r)]
print(f"sanitizer reports: {len(reps)} total, {len(ours)} in simplerecon_b200 code")
for r in ours[:5]:
    print("  ", "; ".join(l.strip() for l in r.splitlines() if re.match(r"\s+#0 ", l))[:300])
PY
    rm -f "$log"
  done
done
