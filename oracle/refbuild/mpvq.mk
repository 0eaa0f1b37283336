# oracle/refbuild/mpvq.mk -- TEST INFRASTRUCTURE.
# The reference's encoder quantisers (libavcodec/mpegvideo_enc.c, UNMODIFIED, read in place and #included by refapi_mpvq.c so that its
# static dct_quantize_trellis_c / denoise_dct_c / clip_coeffs / dct_single_coeff_elimination can be reached) as oracle/_ref/libmpvqref.so.
# Hidden visibility keeps the file's own external names (ff_dct_quantize_c, ff_mpv_encode_init, ...) inside this library; only the
# ref_mpvq_* wrappers are exported.  It links against libavref.so (built first by ./Makefile, whose configuration it shares).
REF   ?= /root/reference
HERE  := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT   := $(abspath $(HERE)/../_ref)
CFG   := $(OUT)/cfg
OBJ   := $(OUT)/obj
CC    ?= gcc
CFLAGS := -O3 -fPIC -std=c99 -fomit-frame-pointer -fno-math-errno -fno-signed-zeros -fno-tree-vectorize \
          -D_ISOC99_SOURCE -D_FILE_OFFSET_BITS=64 -D_LARGEFILE_SOURCE -D_POSIX_C_SOURCE=200112 \
          -D_XOPEN_SOURCE=600 -DHAVE_AV_CONFIG_H -I$(CFG) -I$(REF) -w -fvisibility=hidden

all: $(OUT)/libmpvqref.so

$(OBJ)/mpvq_refapi.o: $(HERE)/refapi_mpvq.c $(REF)/libavcodec/mpegvideo_enc.c $(CFG)/config.h
	$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/libmpvqref.so: $(OBJ)/mpvq_refapi.o $(OUT)/libavref.so
	$(CC) -shared -o $@ $(OBJ)/mpvq_refapi.o -L$(OUT) -lavref -lm -lpthread -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined

.PHONY: all
