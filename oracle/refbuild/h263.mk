# oracle/refbuild/h263.mk -- TEST INFRASTRUCTURE.
# The reference's H.263 deblocking filter (libavcodec/h263dsp.c and libavcodec/h263.c, UNMODIFIED, read in place) with refapi_h263.c
# as oracle/_ref/libh263ref.so.  It links against libavref.so (built first by ./Makefile, whose configuration it shares) for
# ff_init_block_index, av_frame_alloc and the tables h263.c references; nothing else is left unresolved, so no stand-ins are needed.
REF   ?= /root/reference
HERE  := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
OUT   := $(abspath $(HERE)/../_ref)
CFG   := $(OUT)/cfg
OBJ   := $(OUT)/obj
CC    ?= gcc
CFLAGS := -O3 -fPIC -std=c99 -fomit-frame-pointer -fno-math-errno -fno-signed-zeros -fno-tree-vectorize \
          -D_ISOC99_SOURCE -D_FILE_OFFSET_BITS=64 -D_LARGEFILE_SOURCE -D_POSIX_C_SOURCE=200112 \
          -D_XOPEN_SOURCE=600 -DHAVE_AV_CONFIG_H -I$(CFG) -I$(REF) -w
H263_OBJS := $(OBJ)/h263_c_h263dsp.o $(OBJ)/h263_c_h263.o $(OBJ)/h263_refapi.o

all: $(OUT)/libh263ref.so

$(OBJ)/h263_c_%.o: $(REF)/libavcodec/%.c $(CFG)/config.h
	$(CC) $(CFLAGS) -c $< -o $@
$(OBJ)/h263_refapi.o: $(HERE)/refapi_h263.c $(CFG)/config.h
	$(CC) $(CFLAGS) -c $< -o $@

$(OUT)/libh263ref.so: $(H263_OBJS) $(OUT)/libavref.so
	$(CC) -shared -o $@ $(H263_OBJS) -L$(OUT) -lavref -lm -lpthread -Wl,-rpath,'$$ORIGIN' -Wl,--no-undefined

.PHONY: all
