# oracle/haar_dc_stream.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# _ref/libdaala_ref_haar_dc_stream.so: the objects of _ref/libdaala_ref.so (the unmodified reference sources and the
# hook TUs, built by the rules of ./Makefile) plus ref_hooks_haar_dc_stream.c, the DC byte oracle of the engine's
# keyframe DC records (tests/haar_dc_stream_oracle.py).  That TU includes ref_hooks_haar_dc.c, which includes
# src/encode.c, so the TUs that include encode.c too (ref_hooks_encode.c) or call into them (ref_pipeline.c) stay out
# of this library, as in haar_dc.mk.  Needs the reference sources, as `make ref` does:
#   make -C oracle -f haar_dc_stream.mk haar_dc_stream REF=<reference checkout>

include Makefile

.PHONY: haar_dc_stream
haar_dc_stream: $(OUT)/libdaala_ref_haar_dc_stream.so

$(OUT)/c/ref_hooks_haar_dc_stream.o: ref_hooks_haar_dc.c

$(OUT)/libdaala_ref_haar_dc_stream.so: $(filter-out $(OUT)/c/ref_hooks_encode.o $(OUT)/c/ref_pipeline.o,$(C_OBJS)) \
                                       $(OUT)/c/ref_hooks_haar_dc_stream.o
	$(CC) -shared -o $@ $^ -lm
