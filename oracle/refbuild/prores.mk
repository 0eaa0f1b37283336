# oracle/refbuild/prores.mk -- TEST INFRASTRUCTURE.
# oracle/_ref/libproresref.so: the reference's ProRes decoder and encoder, i.e. the UNMODIFIED libavcodec/proresdsp.c, simple_idct.c,
# proresdata.c, and proresdec.c / proresenc.c (#included by refapi_prores.c), linked against libavref.so, which provides the FDCTs,
# the frame, option and pixel-format helpers and av_log.
# The shared configuration has every codec off, so this build takes a copy of it with CONFIG_PRORES_DECODER and CONFIG_PRORES_ENCODER
# set (cfg_prores/), searched before the shared one.  Everything is compiled with hidden visibility: the library exports only the
# ref_prores_* functions of refapi_prores.c, so its simple_idct.c never shadows libavref.so's.
# Every other variable and the satellite link line come from Makefile; libav_b200/build.py runs this after it:
#   make -f prores.mk REF=...
include $(dir $(abspath $(lastword $(MAKEFILE_LIST))))Makefile

.DEFAULT_GOAL := $(OUT)/libproresref.so

CFGP := $(OUT)/cfg_prores
PRORES_CFLAGS := $(subst -I$(CFG),-I$(CFGP) -I$(CFG),$(CFLAGS)) -fvisibility=hidden
PRORES_OBJS := $(OBJ)/pr_proresdsp.o $(OBJ)/pr_simple_idct.o $(OBJ)/pr_proresdata.o $(OBJ)/pr_refapi_prores.o

$(CFGP)/config.h: $(CFG)/config.h
	mkdir -p $(CFGP)
	sed -e '/^#define CONFIG_PRORES_[A-Z]* /d' -e 's/^#endif$$/#define CONFIG_PRORES_DECODER 1\n#define CONFIG_PRORES_ENCODER 1\n#endif/' $< > $@.tmp
	grep -q '^#define CONFIG_PRORES_DECODER 1$$' $@.tmp && grep -q '^#define CONFIG_PRORES_ENCODER 1$$' $@.tmp
	mv $@.tmp $@

$(OBJ)/pr_%.o: $(REF)/libavcodec/%.c $(CFGP)/config.h
	$(CC) $(PRORES_CFLAGS) -c $< -o $@
$(OBJ)/pr_refapi_prores.o: $(HERE)/refapi_prores.c $(REF)/libavcodec/proresdec.c $(REF)/libavcodec/proresenc.c $(CFGP)/config.h
	$(CC) $(PRORES_CFLAGS) -c $< -o $@

$(OUT)/libproresref.so: $(PRORES_OBJS) $(OUT)/libavref.so
	$(SAT_LINK)
