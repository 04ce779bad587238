#!/usr/bin/env bash
# Static evidence for the built library (no GPU needed): per-kernel resource usage and the SASS mnemonics that show which
# memory instructions the walkers compile to.  Usage: tools/sass_summary.sh > profiles/rNN_sass_static.md
set -euo pipefail
cd "$(dirname "$0")/.."
SO=nvidia-resiliency-ext_b200/nvidia_resiliency_ext/checkpointing/b200/_lib/libnvrx_snap.so
echo "# Static SASS / resource summary of libnvrx_snap.so (sm_90a), nvcc $(nvcc --version | grep -o 'V[0-9][0-9.]*' | tail -1)"
echo
echo "## Resource usage (cuobjdump -res-usage): no spills (STACK:0, LOCAL:0) in any walker"
echo
echo '| kernel | REG | static SHARED | STACK | LOCAL |'
echo '|---|---|---|---|---|'
cuobjdump -res-usage "$SO" | awk '/Function/ {name=$2} /REG:/ {gsub(":$","",name); split($0,a," "); r="";s="";st="";l="";
  for(i in a){ if(a[i]~/^REG:/)r=substr(a[i],5); if(a[i]~/^SHARED:/)s=substr(a[i],8); if(a[i]~/^STACK:/)st=substr(a[i],7); if(a[i]~/^LOCAL:/)l=substr(a[i],7)}
  print name, r, s, st, l}' | while read -r name r s st l; do echo "| \`$(echo "$name" | c++filt | sed 's/(.*//')\` | $r | $s | $st | $l |"; done
echo
echo "## SASS mnemonic counts per kernel (cuobjdump -sass)"
echo
echo '| kernel | UBLKCP.S.G (TMA bulk g→s) | UBLKCP.G.S (TMA bulk s→g) | SYNCS (mbarrier) | LDG.E[.NA].128 | STG.E[.NA].128 | LDG.E[.NA].64 | STG.E[.NA].64 | SHFL | F2FP.BF16 (cvt.rn.bf16x2) | LDS (table lookups) |'
echo '|---|---|---|---|---|---|---|---|---|---|---|'
cuobjdump -sass "$SO" | awk '
  /Function :/ { if (name != "") print name, a, b, c, d, e, f, g, h, i, j; name=$3; a=b=c=d=e=f=g=h=i=j=0 }
  /UBLKCP\.S\.G/ {a++} /UBLKCP\.G\.S/ {b++} /SYNCS/ {c++} /LDG\.E(\.[A-Z]+)*\.128/ {d++} /STG\.E(\.[A-Z]+)*\.128/ {e++} /LDG\.E(\.[A-Z]+)*\.64/ {f++} /STG\.E(\.[A-Z]+)*\.64/ {g++} /SHFL/ {h++} /F2FP.*BF16/ {i++} / LDS/ {j++}
  END { if (name != "") print name, a, b, c, d, e, f, g, h, i, j }' | while read -r name a b c d e f g h i j; do
    echo "| \`$(echo "$name" | c++filt | sed 's/(.*//')\` | $a | $b | $c | $d | $e | $f | $g | $h | $i | $j |"; done
echo
echo "Reading: \`walk_*<0>\` = pack (+ optional narrow), \`walk_*<1>\` = scatter (+ optional widen).  In the TMA walkers the bulk tiles move"
echo "only through UBLKCP (no per-thread LDG/STG.128 in the tile loop); the remaining LDG/STG are the ragged-edge, narrow and"
echo "widen paths.  \`.NA\` = no-allocate cache hint (streaming data is not kept in L1).  \`crc_chunks\` (opt-in checksum kernel):"
echo "\`LDG.128\` row loads, \`LDS\` = lookups in the shared-memory operator tables, 64 \`SHFL\` = the unrolled chain over the lanes."
