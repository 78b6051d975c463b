#!/bin/bash
# Build library variants on the GPU machine (same sources, extra -D flags) and run a timing tool against each:
#   bash tools/variant_sweep.sh <tag> k2_variant_timing "AZ_K2_LANES=1 AZ_DEFAULT_K2_BLOCKS=5" "AZ_K2_LANES=2"
# Records and the variant libraries go to variant_out/.
tag=$1; tool=$2; shift; shift
mkdir -p variant_out
out=variant_out/variant_${tool}_$tag.jsonl; : > $out
echo '{"variant": "default"}' >> $out
AZ_TAG=default python tools/$tool.py >> $out 2>> variant_out/variant_${tool}_$tag.err
i=0
for v in "$@"; do
  i=$((i+1)); lib=$PWD/variant_out/libaz_v$i.so
  python -m astroz_b200.build --variant $lib $v > /dev/null 2>> variant_out/variant_${tool}_$tag.err || continue
  echo "{\"variant\": \"$v\"}" >> $out
  ASTROZ_B200_LIB=$lib AZ_TAG="$v" python tools/$tool.py >> $out 2>> variant_out/variant_${tool}_$tag.err
done
cat $out
