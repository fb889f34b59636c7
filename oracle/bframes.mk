# oracle/bframes.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# _ref/libdaala_ref_bframes.so: the objects of _ref/libdaala_ref.so (the unmodified reference sources and the
# hook TUs, built by the rules of ./Makefile) plus ref_hooks_bframes.c, the hooks of the engine's B-frame tests
# (tests/bframe_oracle.py).  Needs the reference sources, as `make ref` does:
#   make -C oracle -f bframes.mk bframes REF=<reference checkout>

include Makefile

.PHONY: bframes
bframes: $(OUT)/libdaala_ref_bframes.so

$(OUT)/libdaala_ref_bframes.so: $(C_OBJS) $(OUT)/c/ref_hooks_bframes.o
	$(CC) -shared -o $@ $^ -lm
