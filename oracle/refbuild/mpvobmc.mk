# oracle/refbuild/mpvobmc.mk -- TEST INFRASTRUCTURE.
# The reference's overlapped block motion compensation (libavcodec/mpegvideo_motion.c, UNMODIFIED, read in place; its ff_mpv_motion
# compiled as ref_real_mpv_motion as in mpvmc.mk) with refapi_mpvobmc.c as oracle/_ref/libmpvobmcref.so, linked against libavref.so.
REF   ?= /root/reference
HERE  := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT   := $(abspath $(HERE)/../_ref)
CFG   := $(OUT)/cfg
OBJ   := $(OUT)/obj
CC    ?= gcc
CFLAGS := -O3 -fPIC -std=c99 -fomit-frame-pointer -fno-math-errno -fno-signed-zeros -fno-tree-vectorize \
          -D_ISOC99_SOURCE -D_FILE_OFFSET_BITS=64 -D_LARGEFILE_SOURCE -D_POSIX_C_SOURCE=200112 \
          -D_XOPEN_SOURCE=600 -DHAVE_AV_CONFIG_H -I$(CFG) -I$(REF) -w

all: $(OUT)/libmpvobmcref.so

$(OBJ)/mpvobmc_c_mpegvideo_motion.o: $(REF)/libavcodec/mpegvideo_motion.c $(CFG)/config.h
	$(CC) $(CFLAGS) -Dff_mpv_motion=ref_real_mpv_motion -c $< -o $@
$(OBJ)/mpvobmc_refapi.o: $(HERE)/refapi_mpvobmc.c $(CFG)/config.h
	$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/libmpvobmcref.so: $(OBJ)/mpvobmc_c_mpegvideo_motion.o $(OBJ)/mpvobmc_refapi.o $(OUT)/libavref.so
	$(CC) -shared -o $@ $(OBJ)/mpvobmc_c_mpegvideo_motion.o $(OBJ)/mpvobmc_refapi.o -L$(OUT) -lavref -lm -lpthread -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined

.PHONY: all
