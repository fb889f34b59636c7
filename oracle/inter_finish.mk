# oracle/inter_finish.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product).
#
# _ref/libdaala_ref_inter_finish.so: the objects of _ref/libdaala_ref.so (the unmodified reference sources and the
# hook TUs, built by the rules of ./Makefile) plus ref_inter_finish.c, the frame driver of the P-frame finishing pass
# bound to the reference (tests/inter_finish_oracle.py).  Needs the reference sources, as `make ref` does:
#   make -C oracle -f inter_finish.mk inter_finish REF=<reference checkout>

include Makefile

.PHONY: inter_finish
inter_finish: $(OUT)/libdaala_ref_inter_finish.so

$(OUT)/c/ref_inter_finish.o: inter_finish_driver.inc

$(OUT)/libdaala_ref_inter_finish.so: $(C_OBJS) $(OUT)/c/ref_inter_finish.o
	$(CC) -shared -o $@ $^ -lm
