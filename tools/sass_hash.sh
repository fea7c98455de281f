#!/bin/bash
# SASS fingerprint of the device objects of libicc_b200.so: md5 of `cuobjdump -sass` with blank address lines removed and the
# path-dependent part of anonymous-namespace symbol names normalised.  Two builds with equal fingerprints run the same device code.
# With -k every kernel body is fingerprinted as well ("  md5  object:kernel"), so that an object that gained kernels, or a kernel that
# became a template instantiation, can be compared kernel by kernel.
# usage: tools/sass_hash.sh [-k] [csrc directory]
per_kernel=0; if [ "$1" = "-k" ]; then per_kernel=1; shift; fi
dir="${1:-$(dirname "$0")/../openimucameracalibrator_b200/csrc}"
sass=$(mktemp); trap 'rm -f "$sass"' EXIT
for f in icc_eval icc_eval_tmem icc_init icc_points icc_solver icc_pose icc_camcal icc_rotinit icc_sew icc_static_imu icc_allan icc_outliers; do
  cuobjdump -sass "$dir/$f.o" | grep -v '^\s*/\*[0-9a-f]\{4\}\*/\s*$' | sed -E 's/_GLOBAL__N__[0-9a-f]+_[0-9]+_[A-Za-z0-9_]+_cu_[0-9a-f]+/_ANON_/g' > "$sass"
  echo "$(md5sum < "$sass" | cut -d' ' -f1)  $f.o"
  if [ "$per_kernel" = 1 ]; then
    awk -v obj="$f.o" '
      /Function : / { if (name != "") close(cmd); name = $NF; cmd = "md5sum | sed \"s|  -$|  " obj ":" name "|; s|^|  |\""; next }
      name != "" { print | cmd }' "$sass"
  fi
done
