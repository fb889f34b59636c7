# oracle/late_skip.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# _ref/libdaala_ref_late_skip.so: the objects of _ref/libdaala_ref.so (the unmodified reference sources and the
# hook TUs, built by the rules of ./Makefile) plus ref_late_skip.c, the late-skip distortion driver bound to the
# reference (tests/late_skip_oracle.py).  Needs the reference sources, as `make ref` does:
#   make -C oracle -f late_skip.mk late_skip REF=<reference checkout>

include Makefile

.PHONY: late_skip
late_skip: $(OUT)/libdaala_ref_late_skip.so

$(OUT)/c/ref_late_skip.o: late_skip_driver.inc

$(OUT)/libdaala_ref_late_skip.so: $(C_OBJS) $(OUT)/c/ref_late_skip.o
	$(CC) -shared -o $@ $^ -lm
