# oracle/refbuild/mpvcf.mk -- TEST INFRASTRUCTURE.
# oracle/_ref/libmpvcfref.so: the motion compensation of MPEG-2 pictures in any chroma format (4:2:0, 4:2:2, 4:4:4), i.e. the UNMODIFIED
# libavcodec/mpegvideo_motion.c -- the same ref_real_mpv_motion object libmpvmcref.so links -- with refapi_mpvcf.c, linked against
# libavref.so, which provides the DSP tables, av_frame_alloc and av_log.
# Every variable, compile rule and the satellite link line come from Makefile; libav_b200/build.py runs this after it:
#   make -f mpvcf.mk REF=...
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.DEFAULT_GOAL := $(OUT)/libmpvcfref.so

$(OUT)/libmpvcfref.so: $(OBJ)/c_mpegvideo_motion.o $(OBJ)/refapi_mpvcf.o $(OUT)/libavref.so
	$(SAT_LINK)
