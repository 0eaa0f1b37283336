# oracle/refbuild/dnxhd_enc.mk -- TEST INFRASTRUCTURE.
# oracle/_ref/libdnxhdencref.so: the reference's VC-3 / DNxHD encoder, i.e. the UNMODIFIED libavcodec/dnxhdenc.c (#included by
# refapi_dnxhd_enc.c) and dnxhddata.c, linked against libavref.so, which provides the DSP inits, the quantiser, the option and frame
# helpers and av_log.  Both compile against the shared configuration, with hidden visibility, so the library exports only the
# ref_dnxhd_* functions of refapi_dnxhd_enc.c and its ff_alloc_packet / av_packet_new_side_data bind locally.
# Every other variable and the satellite link line come from Makefile; libav_b200/build.py runs this after the other satellites:
#   make -f dnxhd_enc.mk REF=...
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.DEFAULT_GOAL := $(OUT)/libdnxhdencref.so

DNXHD_CFLAGS := $(CFLAGS) -fvisibility=hidden

$(OBJ)/dx_dnxhddata.o: $(REF)/libavcodec/dnxhddata.c $(CFG)/config.h
	$(CC) $(DNXHD_CFLAGS) -c $< -o $@
$(OBJ)/dx_refapi_dnxhd_enc.o: $(HERE)/refapi_dnxhd_enc.c $(REF)/libavcodec/dnxhdenc.c $(CFG)/config.h
	$(CC) $(DNXHD_CFLAGS) -c $< -o $@

$(OUT)/libdnxhdencref.so: $(OBJ)/dx_dnxhddata.o $(OBJ)/dx_refapi_dnxhd_enc.o $(OUT)/libavref.so
	$(SAT_LINK)
