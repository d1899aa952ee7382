# Builds oracle/_ref/libflbref_tail.so (tail_harness.c: in_tail's `Parser` branch around the reference's flb_parser_do() and
# log event encoder) with the flags of the reference build, linked against libflbref.so like the shim plugin.
# Run after that Makefile: make -C oracle/refshim -f tail.mk tail.  Test infrastructure only.
include Makefile

tail: $(OUT)/libflbref_tail.so
$(OUT)/libflbref_tail.so: tail_harness.c $(OUT)/libflbref.so
	@$(CC) $(CFLAGS) -shared -o $@ tail_harness.c -L$(OUT) -lflbref -Wl,-rpath,'$$ORIGIN' -Wl,-z,defs -lm
.PHONY: tail
