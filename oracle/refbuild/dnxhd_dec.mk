# oracle/refbuild/dnxhd_dec.mk -- TEST INFRASTRUCTURE.
# oracle/_ref/libdnxhddecref.so: the reference's VC-3 / DNxHD decoder, i.e. the UNMODIFIED libavcodec/dnxhddec.c (#included by
# refapi_dnxhd_dec.c), bitstream.c (init_vlc) and dnxhddata.c, linked against libavref.so, which provides the IDCT and block DSP inits,
# the scan tables, av_reduce, av_image_check_size and av_log.  All compile against the shared configuration with hidden visibility, so the
# library exports only the ref_dnxhd_* functions of refapi_dnxhd_dec.c and its ff_thread_get_buffer / ff_set_dimensions bind locally.
# Every other variable and the satellite link line come from Makefile; libav_b200/build.py runs this after the other satellites:
#   make -f dnxhd_dec.mk REF=...
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.DEFAULT_GOAL := $(OUT)/libdnxhddecref.so

DNXHDDEC_CFLAGS := $(CFLAGS) -fvisibility=hidden

$(OBJ)/dd_%.o: $(REF)/libavcodec/%.c $(CFG)/config.h
	$(CC) $(DNXHDDEC_CFLAGS) -c $< -o $@
$(OBJ)/dd_refapi_dnxhd_dec.o: $(HERE)/refapi_dnxhd_dec.c $(REF)/libavcodec/dnxhddec.c $(CFG)/config.h
	$(CC) $(DNXHDDEC_CFLAGS) -c $< -o $@

$(OUT)/libdnxhddecref.so: $(OBJ)/dd_dnxhddata.o $(OBJ)/dd_bitstream.o $(OBJ)/dd_refapi_dnxhd_dec.o $(OUT)/libavref.so
	$(SAT_LINK)
