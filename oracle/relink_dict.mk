# oracle/relink_dict.mk -- TEST INFRASTRUCTURE ONLY (never linked into the product library).
#
# _ref/relinked_dict: the reference's UNMODIFIED frame layer (lib/lizard_frame.c + lib/xxhash/xxhash.c, compiled from
# the sources where they lie under $(REF)) linked against ../lizard_b200/liblizard_b200.so, with oracle/relink_dict_main.c as
# its main: a frame of linked blocks then decodes through our Lizard_decompress_safe_usingDict (tests/test_gpu_dict.py).
# Built next to the binaries of Makefile's `ref` target (whose REF and CC it takes), under the same condition as its
# relinked_frame: the reference tree and the library are both present.  Nothing is copied; the output goes only to
# oracle/_ref/ (git-ignored).
#
#   make -C oracle -f relink_dict.mk
include Makefile
.DEFAULT_GOAL := relinked_dict

relinked_dict:
	@if [ -d $(REF)/lib ] && [ -f ../lizard_b200/liblizard_b200.so ]; then \
	  mkdir -p _ref && \
	  $(CC) -O2 -w -I$(REF)/lib -DXXH_NAMESPACE=Lizard_ -o _ref/relinked_dict relink_dict_main.c \
	    $(REF)/lib/lizard_frame.c $(REF)/lib/xxhash/xxhash.c \
	    -L../lizard_b200 -llizard_b200 -Wl,-rpath,'$$ORIGIN/../../lizard_b200' -lm && \
	  echo "oracle/_ref/relinked_dict built from $(REF)"; \
	else echo "reference tree $(REF) or the library absent: using a prebuilt oracle/_ref/relinked_dict if any"; fi
.PHONY: relinked_dict
