# oracle/refbuild/xvid.mk -- TEST INFRASTRUCTURE.
# The reference's Xvid IDCT (libavcodec/xvididct.c, UNMODIFIED, read in place) with refapi_xvid.c as oracle/_ref/libxvidref.so.  It links
# against libavref.so (built first by ./Makefile, whose configuration it shares) for ff_idctdsp_init and the pixel helpers.  The x86 hook
# ff_xvid_idct_init_x86 is compiled out: the shared configuration has ARCH_X86 0.
REF   ?= /root/reference
HERE  := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT   := $(abspath $(HERE)/../_ref)
CFG   := $(OUT)/cfg
OBJ   := $(OUT)/obj
CC    ?= gcc
CFLAGS := -O3 -fPIC -std=c99 -fomit-frame-pointer -fno-math-errno -fno-signed-zeros -fno-tree-vectorize \
          -D_ISOC99_SOURCE -D_FILE_OFFSET_BITS=64 -D_LARGEFILE_SOURCE -D_POSIX_C_SOURCE=200112 \
          -D_XOPEN_SOURCE=600 -DHAVE_AV_CONFIG_H -I$(CFG) -I$(REF) -w

all: $(OUT)/libxvidref.so

$(OBJ)/xvid_c_xvididct.o: $(REF)/libavcodec/xvididct.c $(CFG)/config.h
	$(CC) $(CFLAGS) -c $< -o $@
$(OBJ)/xvid_refapi.o: $(HERE)/refapi_xvid.c $(CFG)/config.h
	$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/libxvidref.so: $(OBJ)/xvid_c_xvididct.o $(OBJ)/xvid_refapi.o $(OUT)/libavref.so
	$(CC) -shared -o $@ $(OBJ)/xvid_c_xvididct.o $(OBJ)/xvid_refapi.o -L$(OUT) -lavref -lm -lpthread -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined

.PHONY: all
