# oracle/lossless.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# _ref/libdaala_ref_lossless.so: the objects of _ref/libdaala_ref.so (the unmodified reference sources and the hook
# TUs, built by the rules of ./Makefile) plus ref_hooks_lossless.c, the quantizer-0 frame driver of the engine's
# lossless tests (tests/lossless_oracle.py).  ref_hooks_lossless.c includes src/encode.c as ref_hooks_encode.c does,
# so that TU, and ref_pipeline.c which calls into it, stay out of this library.  Needs the reference sources, as
# `make ref` does:
#   make -C oracle -f lossless.mk lossless REF=<reference checkout>

include Makefile

.PHONY: lossless
lossless: $(OUT)/libdaala_ref_lossless.so

$(OUT)/libdaala_ref_lossless.so: $(filter-out $(OUT)/c/ref_hooks_encode.o $(OUT)/c/ref_pipeline.o,$(C_OBJS)) \
                                 $(OUT)/c/ref_hooks_lossless.o
	$(CC) -shared -o $@ $^ -lm
