#!/bin/bash
# CPU stand-ins for compute-sanitizer on the SIMT kernels (tests/emul: one host thread per CUDA thread, real barriers):
#   memcheck  -> AddressSanitizer + UBSan build of the emulated kernels (out-of-bounds shared / global accesses, misaligned
#                vector loads, signed overflow in index math)
#   racecheck -> ThreadSanitizer build (a missing __syncthreads / __syncwarp between a shared-memory write and another
#                thread's read is a data race); reports whose frames are all inside torch / libgomp are artefacts of the
#                un-instrumented interpreter — only frames under deepinv_b200/csrc matter.
# usage: tools/sanitize_emul.sh [memcheck|racecheck] [pytest args...]
set -u
MODE=${1:-memcheck}; shift || true
TESTS=${*:-tests/test_emul_kernels.py tests/test_random_shapes_emul.py tests/test_edge_cases_emul.py tests/test_emul_pipe_kernels.py tests/test_emul_tc32_simt.py tests/test_host_logic_emul.py tests/test_emul_svblur.py tests/test_emul_tv.py tests/test_emul_tgv.py tests/test_emul_spectral_paths.py tests/test_emul_tiledsv.py tests/test_emul_radon_paths.py tests/test_emul_blur_paths.py tests/test_emul_blur3d_paths.py tests/test_emul_mri3d_paths.py tests/test_emul_conv3d.py tests/test_emul_resize.py}
if [ "$MODE" = "racecheck" ]; then
  rm -f /tmp/dinvk_tsan.*
  DINVK_EMUL_SANITIZE=thread LD_PRELOAD=$(gcc -print-file-name=libtsan.so) \
    TSAN_OPTIONS="halt_on_error=0 report_signal_unsafe=0 log_path=/tmp/dinvk_tsan history_size=4" python -m pytest $TESTS -x -q | tail -3
  echo "TSan reports with kernel frames (must be empty):"
  grep -h "csrc/" /tmp/dinvk_tsan.* 2>/dev/null | grep -v "spectral.cu:[0-9]* *$" | sort | uniq -c | sort -rn | head -20
else
  DINVK_EMUL_SANITIZE=1 LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 \
    UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=1 python -m pytest $TESTS -x -q | tail -3
fi
