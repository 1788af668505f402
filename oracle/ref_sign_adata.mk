# oracle/ref_sign_adata.mk — builds oracle/_ref/libecc_ref_sign_adata.so: the reference's ECKCDSA / ECGDSA / ECRDSA /
# SM2 signer with injected nonces and per-item ancillary data, and ec_verify with that data (ref_sign_adata.c), linked
# to the unmodified reference oracle/Makefile builds.  TEST INFRASTRUCTURE, like that file.
# Only built where the reference's sources lie under $(REF); elsewhere the prebuilt library is used.
#
#   make -C oracle -f ref_sign_adata.mk        (after make -C oracle ref)

REF ?= /root/reference
OUT := _ref
CC  ?= gcc

all: $(if $(wildcard $(REF)/src/libsig.h),$(OUT)/libecc_ref_sign_adata.so,)

$(OUT)/libecc_ref_sign_adata.so: ref_sign_adata.c $(OUT)/libecc_ref.so
	$(CC) -O2 -std=gnu11 -fPIC -shared -DWITH_STDLIB -w -I$(REF)/src $< -o $@ -L$(OUT) -lecc_ref -Wl,-rpath,'$$ORIGIN' -lpthread

.PHONY: all
