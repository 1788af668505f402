# oracle/ref_bign.mk — builds oracle/_ref/libecc_ref_bign.so: the reference's BIGN / DBIGN signer with injected nonces
# and per-item adata records, its BIGN ec_verify, and its BELT / BASH primitives (ref_bign.c), linked to the
# unmodified reference oracle/Makefile builds.  TEST INFRASTRUCTURE, like that file.
# Only built where the reference's sources lie under $(REF); elsewhere the prebuilt library is used.
#
#   make -C oracle -f ref_bign.mk        (after make -C oracle ref)

REF ?= /root/reference
OUT := _ref
CC  ?= gcc

all: $(if $(wildcard $(REF)/src/libsig.h),$(OUT)/libecc_ref_bign.so,)

$(OUT)/libecc_ref_bign.so: ref_bign.c $(OUT)/libecc_ref.so
	$(CC) -O2 -std=gnu11 -fPIC -shared -DWITH_STDLIB -w -I$(REF)/src $< -o $@ -L$(OUT) -lecc_ref -Wl,-rpath,'$$ORIGIN' -lpthread

.PHONY: all
