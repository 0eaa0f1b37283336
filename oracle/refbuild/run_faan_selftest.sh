#!/bin/sh
# Builds the reference's own DCT self test (libavcodec/tests/dct.c) against oracle/_ref/libavref.so and records, for tests 0 / 1 / 2, its
# 'IDCT FAANI' lines (ff_faanidct, `dct -i <test>`) as known answers in tests/golden/fate_dct8x8_faan.txt.  Run where the reference tree is; the output file is committed.
set -e
HERE=$(cd "$(dirname "$0")" && pwd); ROOT=$(cd "$HERE/../.." && pwd); REF=${REF:-/root/reference}
OUT=$ROOT/oracle/_ref
make -s -C "$HERE" REF="$REF"
gcc -O2 -std=c99 -D_ISOC99_SOURCE -D_POSIX_C_SOURCE=200112 -D_XOPEN_SOURCE=600 -DHAVE_AV_CONFIG_H \
    -I"$OUT/cfg" -I"$REF" -w -o "$OUT/dct_selftest_faan" "$REF/libavcodec/tests/dct.c" "$REF/libavcodec/dctref.c" \
    "$REF/libavcodec/aandcttab.c" "$REF/libavcodec/xvididct.c" -L"$OUT" -lavref -lm -Wl,-rpath,"$OUT"
G=$ROOT/tests/golden/fate_dct8x8_faan.txt
echo "# libavcodec/tests/dct -i <test>: the 'IDCT FAANI' line (NB_ITS=20000, av_lfg seed 1)" > "$G"
for t in 0 1 2; do
    "$OUT/dct_selftest_faan" -i $t | grep '^IDCT FAANI:' | sed "s/^IDCT FAANI:/idct$t/" >> "$G"
done
cat "$G"
