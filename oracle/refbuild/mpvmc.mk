# oracle/refbuild/mpvmc.mk -- TEST INFRASTRUCTURE.
# The reference's motion compensation for the mpegvideo decoders (libavcodec/mpegvideo_motion.c, UNMODIFIED, read in place) with
# refapi_mpvmc.c as oracle/_ref/libmpvmcref.so.  It links against libavref.so (built first by ./Makefile, whose configuration it shares)
# for ff_hpeldsp_init, ff_qpeldsp_init, ff_videodsp_init, av_frame_alloc and av_log.  libavref.so already exports an aborting stand-in
# named ff_mpv_motion (refapi_mpv_stubs.c): the real function is compiled under the name ref_real_mpv_motion so that the two never meet.
REF   ?= /root/reference
HERE  := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT   := $(abspath $(HERE)/../_ref)
CFG   := $(OUT)/cfg
OBJ   := $(OUT)/obj
CC    ?= gcc
CFLAGS := -O3 -fPIC -std=c99 -fomit-frame-pointer -fno-math-errno -fno-signed-zeros -fno-tree-vectorize \
          -D_ISOC99_SOURCE -D_FILE_OFFSET_BITS=64 -D_LARGEFILE_SOURCE -D_POSIX_C_SOURCE=200112 \
          -D_XOPEN_SOURCE=600 -DHAVE_AV_CONFIG_H -I$(CFG) -I$(REF) -w

all: $(OUT)/libmpvmcref.so

$(OBJ)/mpvmc_c_mpegvideo_motion.o: $(REF)/libavcodec/mpegvideo_motion.c $(CFG)/config.h
	$(CC) $(CFLAGS) -Dff_mpv_motion=ref_real_mpv_motion -c $< -o $@
$(OBJ)/mpvmc_refapi.o: $(HERE)/refapi_mpvmc.c $(CFG)/config.h
	$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/libmpvmcref.so: $(OBJ)/mpvmc_c_mpegvideo_motion.o $(OBJ)/mpvmc_refapi.o $(OUT)/libavref.so
	$(CC) -shared -o $@ $(OBJ)/mpvmc_c_mpegvideo_motion.o $(OBJ)/mpvmc_refapi.o -L$(OUT) -lavref -lm -lpthread -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined

.PHONY: all
