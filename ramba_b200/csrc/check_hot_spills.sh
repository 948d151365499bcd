#!/bin/bash
# Static check of the 1-D kernel after a build: local-memory (spill) instructions and register shuffles in the tile
# loop and the dispatch loop.  ptxas runs this kernel at the 128-register cap; small source changes decide whether
# loop-carried state stays in registers.  usage: check_hot_spills.sh build/rb200_elementwise_nd1.o
o=$1
cuobjdump -sass -fun '_ZN5rb20021vm_elementwise_kernelILi8ELi1ELb0ELb0EEEvNS_7KParamsE' $o | grep -E "^\s+/\*[0-9a-f]{4,}\*/" | sed 's/\/\* 0x[0-9a-f]* \*\///' > /tmp/hs.sass
total=$(wc -l < /tmp/hs.sass)
h=$(grep -n "LDCU\?\.U16" /tmp/hs.sass | head -1 | cut -d: -f1)  # the load of the handler id opens the dispatch loop
echo "total instrs $total; LDL/STL total $(grep -c 'LDL\|STL' /tmp/hs.sass); handler-load line $h"
echo "tile loop + dispatch head (lines 1..$((h+60))):"; head -$((h+60)) /tmp/hs.sass | grep -n "LDL\|STL" | awk '{print $1,$3,$4,$5}' | tr '\n' ';'; echo
echo "MOVs between handler load and +45: $(sed -n "$h,$((h+45))p" /tmp/hs.sass | grep -c 'MOV')"
n=$(grep -n "c\[0x0\]\[0x384\]" /tmp/hs.sass | tail -1 | cut -d: -f1)
echo "latch region LDL/STL: $(sed -n "$((n-12)),$((n+12))p" /tmp/hs.sass | grep -c 'LDL\|STL')"
