#!/bin/bash
# Opcode mix of the headline pass kernels in the built library (run after a build): registers / spills from ptxas -v,
# instruction counts per opcode from cuobjdump -sass, and the TMA / mbarrier / FP64-quotient mnemonics that prove the design.
cd "$(dirname "$0")/.."
LIB=${1:-fastecc_b200/libfastecc_b200.so}
cuobjdump -sass $LIB > /tmp/all.sass
echo "# $LIB  ($(cuobjdump -lelf $LIB | grep -c sm_90a) sm_90a cubins)"
for pat in "pass_kernelILi10ELi2ELi1" "pass_kernelILi9ELi1ELi1" "pass_kernelILi9ELi1ELi2" "pass_kernelILi10ELi2ELi2"; do
  s=$(grep -n "Function : .*${pat}" /tmp/all.sass | cut -d: -f1)
  [ -z "$s" ] && continue
  e=$(awk -v s=$s 'NR>s && /Function :/{print NR; exit}' /tmp/all.sass); [ -z "$e" ] && e=$(wc -l < /tmp/all.sass)
  sed -n "${s},${e}p" /tmp/all.sass | grep -E "^\s+/\*[0-9a-f]{4,5}\*/" | sed 's/\/\*[0-9a-f]*\*\/\s*$//' | awk '{ $1=""; print}' | sed 's/\/\*.*//' > /tmp/k.sass
  echo "== ntt_pass_kernel<$(echo $pat | sed 's/pass_kernelILi//; s/ELi/,/g')>: $(wc -l < /tmp/k.sass) instructions; LDL/STL $(grep -c -E 'LDL|STL' /tmp/k.sass); IMAD.HI $(grep -c IMAD.HI /tmp/k.sass)"
  awk '{ if ($1 ~ /^@/) print $2; else print $1}' /tmp/k.sass | sed 's/;//' | sort | uniq -c | sort -rn | head -28 | awk '{printf "%6d %-22s", $1, $2; if (NR % 4 == 0) printf "\n"} END {printf "\n"}'
done
echo "== whole library: UTMALDG $(grep -c UTMALDG /tmp/all.sass)  UBLKCP $(grep -c UBLKCP /tmp/all.sass)  SYNCS $(grep -c 'SYNCS' /tmp/all.sass)  I2F.F64.U32 $(grep -c 'I2F.F64.U32' /tmp/all.sass)  DFMA.RM $(grep -c 'DFMA.RM' /tmp/all.sass)  VIADDMNMX.U32 $(grep -c 'VIADDMNMX.U32' /tmp/all.sass)"
