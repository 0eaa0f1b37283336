#!/bin/sh
# Builds the reference's own IDCT self test (libavcodec/tests/dct.c, FATE target fate-idct8x8) with its XVID row and records the
# 'IDCT XVID' lines as known answers in tests/golden/fate_idct8x8_xvid.txt.  dct.c compiles that row only when CONFIG_MPEG4_DECODER is
# set, so the test is built against a copy of oracle/_ref/cfg that differs in that one macro.  The same binary's SIMPLE-C lines equal
# tests/golden/fate_idct8x8.txt.  Run where the reference tree is; the output file is committed.
set -e
HERE=$(cd "$(dirname "$0")" && pwd); ROOT=$(cd "$HERE/../.." && pwd); REF=${REF:-/root/reference}
OUT=$ROOT/oracle/_ref
make -s -C "$HERE" REF="$REF"
rm -rf "$OUT/cfg_mpeg4"; mkdir -p "$OUT/cfg_mpeg4"; cp -r "$OUT/cfg/." "$OUT/cfg_mpeg4/"
sed -i 's/^#define CONFIG_MPEG4_DECODER 0$/#define CONFIG_MPEG4_DECODER 1/' "$OUT/cfg_mpeg4/config.h"
grep -q '^#define CONFIG_MPEG4_DECODER 1$' "$OUT/cfg_mpeg4/config.h"
gcc -O2 -std=c99 -D_ISOC99_SOURCE -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -DHAVE_AV_CONFIG_H \
    -I"$OUT/cfg_mpeg4" -I"$REF" -w -o "$OUT/dct_selftest_xvid" "$REF/libavcodec/tests/dct.c" "$REF/libavcodec/dctref.c" \
    "$REF/libavcodec/aandcttab.c" "$REF/libavcodec/xvididct.c" -L"$OUT" -lavref -lm -Wl,-rpath,"$OUT"
G=$ROOT/tests/golden/fate_idct8x8_xvid.txt
echo "# libavcodec/tests/dct -i <test>: the 'IDCT XVID' line (NB_ITS=20000, av_lfg seed 1; built with CONFIG_MPEG4_DECODER 1)" > "$G"
for t in 0 1 2; do
    "$OUT/dct_selftest_xvid" -i $t | grep 'IDCT XVID' | sed "s/^IDCT XVID:/test$t/" >> "$G"
done
cat "$G"
