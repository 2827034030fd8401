# oracle/alpha_probe.mk -- TEST INFRASTRUCTURE, not product code: builds oracle/_ref/alpha_probe
# (probe/alpha_probe.cpp) against the unmodified reference library that oracle/Makefile builds, with its flags.
# `make -f alpha_probe.mk` after `make ref`; skipped where the reference sources are absent.
include Makefile

$(OUT)/alpha_probe: $(OBJ)/probe/alpha_probe.o $(OUT)/libpbrt_ref.a
	$(CXX) -o $@ $< $(OUT)/libpbrt_ref.a -lpthread

alpha_probe:
	@if [ -d $(REF)/src ]; then $(MAKE) -f alpha_probe.mk $(OUT)/alpha_probe; else echo "no $(REF): keeping prebuilt _ref"; fi
.PHONY: alpha_probe
