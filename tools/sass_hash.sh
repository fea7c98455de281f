#!/bin/bash
# SASS fingerprint of the device objects of libicc_b200.so: md5 of `cuobjdump -sass` with blank address lines removed and the
# path-dependent part of anonymous-namespace symbol names normalised.  Two builds with equal fingerprints run the same device code.
# usage: tools/sass_hash.sh [csrc directory]
dir="${1:-$(dirname "$0")/../openimucameracalibrator_b200/csrc}"
for f in icc_eval icc_eval_tmem icc_init icc_points icc_solver icc_pose icc_camcal icc_rotinit icc_sew icc_static_imu icc_allan; do
  h=$(cuobjdump -sass "$dir/$f.o" | grep -v '^\s*/\*[0-9a-f]\{4\}\*/\s*$' | sed -E 's/_GLOBAL__N__[0-9a-f]+_[0-9]+_[A-Za-z0-9_]+_cu_[0-9a-f]+/_ANON_/g' | md5sum | cut -d' ' -f1)
  echo "$h  $f.o"
done
