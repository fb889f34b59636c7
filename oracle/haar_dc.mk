# oracle/haar_dc.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# _ref/libdaala_ref_haar_dc.so: the objects of _ref/libdaala_ref.so (the unmodified reference sources and the hook
# TUs, built by the rules of ./Makefile) plus ref_hooks_haar_dc.c, the keyframe DC driver of the engine's
# haar_dc_quant tests (tests/haar_dc_oracle.py).  ref_hooks_haar_dc.c includes src/encode.c as ref_hooks_encode.c
# does, so that TU, and ref_pipeline.c which calls into it, stay out of this library.  Needs the reference sources, as
# `make ref` does:
#   make -C oracle -f haar_dc.mk haar_dc REF=<reference checkout>

include Makefile

.PHONY: haar_dc
haar_dc: $(OUT)/libdaala_ref_haar_dc.so

$(OUT)/libdaala_ref_haar_dc.so: $(filter-out $(OUT)/c/ref_hooks_encode.o $(OUT)/c/ref_pipeline.o,$(C_OBJS)) \
                                $(OUT)/c/ref_hooks_haar_dc.o
	$(CC) -shared -o $@ $^ -lm
