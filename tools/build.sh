#!/bin/bash
# Rebuild the product library (sm_90a) and the test-only host shim; prints ptxas resource lines.
set -e
R="$(cd "$(dirname "$0")/.." && pwd)"
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -shared -Xlinker -Bsymbolic-functions -Xptxas -v \
     -o "$R/lizard_b200/liblizard_b200.so" "$R/lizard_b200/csrc/api.cu" 2>&1 | grep -E "error|warning|Compiling|registers|spill" || true
# the encode kernel's instances (ILi0E Fast = levels 10/11, ILi1E FastBig = 20, ILi2E Generic = the rest)
cuobjdump -res-usage "$R/lizard_b200/liblizard_b200.so" | grep -A1 lizard_encode_units_kernel || true
g++ -O2 -fPIC -shared -x c++ -std=c++17 -o "$R/lizard_b200/libhostshim.so" "$R/lizard_b200/csrc/host_shim.cpp"
