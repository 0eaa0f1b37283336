# oracle/refbuild/prores_enc.mk -- TEST INFRASTRUCTURE.
# oracle/_ref/libproresencref.so: the reference's ProRes encoder with every option, i.e. the UNMODIFIED libavcodec/proresenc.c
# (#included by refapi_prores_enc.c) and proresdata.c, linked against libavref.so, which provides the FDCTs, the frame, option and
# pixel-format helpers and av_log.  The configuration, flags and the proresdata.c object are prores.mk's; everything is compiled with
# hidden visibility, so the library exports only the ref_prores_enc* functions of refapi_prores_enc.c.
# libav_b200/build.py runs this after prores.mk:
#   make -f prores_enc.mk REF=...
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))prores.mk

.DEFAULT_GOAL := $(OUT)/libproresencref.so

$(OBJ)/pr_refapi_prores_enc.o: $(HERE)/refapi_prores_enc.c $(REF)/libavcodec/proresenc.c $(CFGP)/config.h
	$(CC) $(PRORES_CFLAGS) -c $< -o $@

$(OUT)/libproresencref.so: $(OBJ)/pr_proresdata.o $(OBJ)/pr_refapi_prores_enc.o $(OUT)/libavref.so
	$(SAT_LINK)
