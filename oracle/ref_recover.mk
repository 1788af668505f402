# oracle/ref_recover.mk — builds oracle/_ref/libecc_ref_recover.so: the reference's ECDSA public-key recovery and its
# y-from-x lift (ref_recover.c), linked to the unmodified reference oracle/Makefile builds.  TEST INFRASTRUCTURE, like
# that file.  Only built where the reference's sources lie under $(REF); elsewhere the prebuilt library is used.
#
#   make -C oracle -f ref_recover.mk        (after make -C oracle ref)

REF ?= /root/reference
OUT := _ref
CC  ?= gcc

all: $(if $(wildcard $(REF)/src/libsig.h),$(OUT)/libecc_ref_recover.so,)

$(OUT)/libecc_ref_recover.so: ref_recover.c $(OUT)/libecc_ref.so
	$(CC) -O2 -std=gnu11 -fPIC -shared -DWITH_STDLIB -w -I$(REF)/src $< -o $@ -L$(OUT) -lecc_ref -Wl,-rpath,'$$ORIGIN'

.PHONY: all
