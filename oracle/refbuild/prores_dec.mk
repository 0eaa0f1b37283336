# oracle/refbuild/prores_dec.mk -- TEST INFRASTRUCTURE.
# oracle/_ref/libproresdecref.so: the reference's ProRes decoder with the checked bitstream reader, i.e. the UNMODIFIED
# libavcodec/proresdec.c (#included by refapi_prores_dec.c, which selects the checked reader) beside prores.mk's proresdsp.c, simple_idct.c
# and proresdata.c objects, linked against libavref.so, which provides the scan-table init, the frame and pixel-format helpers and av_log.
# The configuration and flags are prores.mk's; everything is compiled with hidden visibility, so the library exports only the
# ref_prores_dec_* functions of refapi_prores_dec.c.  libav_b200/build.py runs this after prores.mk:
#   make -f prores_dec.mk REF=...
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))prores.mk

.DEFAULT_GOAL := $(OUT)/libproresdecref.so

$(OBJ)/pr_refapi_prores_dec.o: $(HERE)/refapi_prores_dec.c $(REF)/libavcodec/proresdec.c $(CFGP)/config.h
	$(CC) $(PRORES_CFLAGS) -c $< -o $@

$(OUT)/libproresdecref.so: $(OBJ)/pr_proresdsp.o $(OBJ)/pr_simple_idct.o $(OBJ)/pr_proresdata.o $(OBJ)/pr_refapi_prores_dec.o $(OUT)/libavref.so
	$(SAT_LINK)
