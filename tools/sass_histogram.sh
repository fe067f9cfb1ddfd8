#!/bin/bash
# SASS instruction histogram of every kernel in libwhisper_b200.so: the mnemonics that prove the Hopper-native paths
# (HGMMA = wgmma.mma_async, UTMALDG = TMA tile load, UBLKCP = bulk copy, HMMA = mma.sync, SYNCS = mbarrier).
#   usage: tools/sass_histogram.sh > <name>_sass_histogram.txt
SO="$(dirname "$0")/../whisper_b200/libwhisper_b200.so"
cuobjdump -sass "$SO" | awk '
  /Function :/ { name=$3; next }
  /^[ \t]*\/\*[0-9a-f]+\*\// { n[name]++; m=$2; sub(/\..*/,"",m); if (m ~ /^@/) { m=$3; sub(/\..*/,"",m) }
    if (m ~ /^(HGMMA|WARPGROUP|UTMALDG|UTMASTG|UBLKCP|UBLKPF|HMMA|SYNCS|MUFU|LDGSTS|ATOM|RED|BAR|MEMBAR|CCTL|FFMA|F2FP|HADD2|LDS|LDG|STG|STS)$/) c[name" "m]++ }
  END { for (k in n) { printf "%-110s %6d instr :", k, n[k]; for (x in c) { split(x, p, " "); if (p[1]==k) printf " %s=%d", p[2], c[x] } printf "\n" } }' | sort
