#!/bin/bash
# Per-kernel counts of the SASS mnemonics that prove the Hopper paths (wgmma = HGMMA, TMA load/store = UTMALDG/UTMASTG,
# mbarrier = SYNCS, cluster barrier = UCGABAR) and of the legacy HMMA (mma.sync), which must stay at zero:
#   scripts/sass_counts.sh
cd "$(dirname "$0")/.."
SO=stable-diffusion_b200/csrc/libsdb200.so
echo "# cuobjdump -sass $SO  (built $(date -u -r $SO +%Y-%m-%dT%H:%MZ)); counts summed over all template instantiations of a kernel"
cuobjdump -sass $SO | awk '
  /Function :/ { name=$3; sub(/^_ZN3sdb[0-9]*/, "", name); sub(/I[LE].*$/, "", name); sub(/E[0-9A-Za-z_]*$/, "", name); next }
  { for (i = 1; i <= NF; ++i) if ($i ~ /^(HGMMA|UTMALDG|UTMASTG|SYNCS|UCGABAR|HMMA|MUFU)/) { split($i, a, "[._]"); c[name, a[1]]++; k[name]=1 } }
  END { for (n in k) { printf "%-34s", n; split("HGMMA UTMALDG UTMASTG SYNCS UCGABAR MUFU HMMA", m, " "); for (j = 1; j <= 7; ++j) printf " %s=%d", m[j], c[n, m[j]] + 0; printf "\n" } }' | sort
