# Builds oracle/_ref/libflbref_gelf.so: the UNMODIFIED $(REF)/src/flb_pack_gelf.c (not part of libflbref.so) and
# gelf_harness.c (out_gelf's / out_http's flush loop around it), with the flags of the reference build, linked against
# libflbref.so like the shim plugin.  Run after that Makefile: make -C oracle/refshim -f gelf.mk gelf.  Test infrastructure only.
include Makefile

gelf: $(OUT)/libflbref_gelf.so
$(OUT)/libflbref_gelf.so: gelf_harness.c $(REF)/src/flb_pack_gelf.c $(OUT)/libflbref.so
	@$(CC) $(CFLAGS) -shared -o $@ gelf_harness.c $(REF)/src/flb_pack_gelf.c -L$(OUT) -lflbref -Wl,-rpath,'$$ORIGIN' -Wl,-z,defs -lm
.PHONY: gelf
