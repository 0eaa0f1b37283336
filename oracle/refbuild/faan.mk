# oracle/refbuild/faan.mk -- TEST INFRASTRUCTURE.
# The reference's encoder paths behind the FAAN forward DCT (FF_DCT_FAAN), as two satellites linked against libavref.so (which holds
# ff_faandct / ff_faanidct themselves):
#   oracle/_ref/libfaanqref.so    refapi_faanq.c: the quantisers of refapi_mpvq.c (mpegvideo_enc.c, unmodified) with s->fdsp.fdct = ff_faandct
#   oracle/_ref/libfaanencref.so  refapi_faanenc.c: quant_psnr / bit / rd of refapi_enc.c on contexts with s->fdsp.fdct = ff_faandct
# Every variable, compile rule and the satellite link line come from Makefile; libav_b200/build.py runs this after it:
#   make -f faan.mk REF=...
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.DEFAULT_GOAL := faan
.PHONY: faan
faan: $(OUT)/libfaanqref.so $(OUT)/libfaanencref.so

$(OBJ)/refapi_faanq.o: CFLAGS += -fvisibility=hidden
$(OBJ)/refapi_faanq.o: $(REF)/libavcodec/mpegvideo_enc.c $(HERE)/refapi_mpvq.c
$(OBJ)/refapi_faanenc.o: $(HERE)/refapi_enc.c

$(OUT)/libfaanqref.so: $(OBJ)/refapi_faanq.o $(OUT)/libavref.so
	$(SAT_LINK)
$(OUT)/libfaanencref.so: $(OBJ)/refapi_faanenc.o $(OUT)/libavref.so
	$(SAT_LINK)
