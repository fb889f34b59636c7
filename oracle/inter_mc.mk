# oracle/inter_mc.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# _ref/libdaala_ref_inter_mc.so: the objects of _ref/libdaala_ref.so (the unmodified reference sources and the
# hook TUs, built by the rules of ./Makefile) plus ref_hooks_inter_mc.c, the hooks of the engine's P-frame
# prediction tests (tests/inter_mc_oracle.py).  Needs the reference sources, as `make ref` does:
#   make -C oracle -f inter_mc.mk inter_mc REF=<reference checkout>

include Makefile

.PHONY: inter_mc
inter_mc: $(OUT)/libdaala_ref_inter_mc.so

$(OUT)/libdaala_ref_inter_mc.so: $(C_OBJS) $(OUT)/c/ref_hooks_inter_mc.o
	$(CC) -shared -o $@ $^ -lm
