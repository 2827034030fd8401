# nvcc flags of the product build, shared with test harnesses that must compile the device headers exactly as the
# product does (tests/devmath/Makefile).  Set NVCC and EXTRA before including this file.
# -fmad=false: the path's arithmetic must round exactly like the reference's
# scalar float code (no FMA contraction); see DESIGN.md "Numerics".
NVFLAGS := -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -fmad=false \
  -Xcompiler -fPIC,-O3,-ffp-contract=off -Xptxas -v --expt-relaxed-constexpr $(EXTRA)
