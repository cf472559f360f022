#!/bin/bash
# Times the main workloads against each kernel build variant (fundsp_b200/variants/*.so) and the product library.
# usage (on a GPU machine): tools/variant_bench.sh
for lib in fundsp_b200/libfundsp_b200.so fundsp_b200/variants/*.so; do
  [ -f "$lib" ] || continue
  echo "== $lib"
  for w in "saw_svf 16384 mix" "saw_svf 16384 voices" "noise_svf 16384 mix" "fm 4096 mix" "net 65536 mix" "biquad_bank 2048 mix" "subtractive_dry 1024 mix" "subtractive 1024 mix"; do
    set -- $w
    FDSP_B200_LIB=$PWD/$lib python tools/prof_bank.py --workload $1 --voices $2 --mode $3 --n 16384 --iters 3 2>&1 | tail -1
  done
done
