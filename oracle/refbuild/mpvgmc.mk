# oracle/refbuild/mpvgmc.mk -- TEST INFRASTRUCTURE.
# oracle/_ref/libmpvgmcref.so: the motion compensation of MPEG-4 S-VOPs (global motion compensation), i.e. the UNMODIFIED
# libavcodec/mpegvideo_motion.c -- the same ref_real_mpv_motion object libmpvmcref.so links -- with refapi_mpvgmc.c, linked against
# libavref.so, which provides ff_mpegvideodsp_init (gmc1_c, ff_gmc_c), the other DSP tables, av_frame_alloc and av_log.
# Every variable, compile rule and the satellite link line come from Makefile; libav_b200/build.py runs this after it:
#   make -f mpvgmc.mk REF=...
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.DEFAULT_GOAL := $(OUT)/libmpvgmcref.so

$(OUT)/libmpvgmcref.so: $(OBJ)/c_mpegvideo_motion.o $(OBJ)/refapi_mpvgmc.o $(OUT)/libavref.so
	$(SAT_LINK)
