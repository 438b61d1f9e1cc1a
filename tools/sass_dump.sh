#!/bin/bash
# usage: tools/sass_dump.sh [object] [out]   -- line-annotated SASS of the sm_90a cubin inside an object file
obj=${1:-porepy_b200/_obj/libporeb200.so/mpsa3d.o}; out=${2:-/tmp/api.sass}
tmp=$(mktemp -d); ( cd $tmp && cuobjdump -xelf all "$OLDPWD/$obj" > /dev/null )
nvdisasm -g $tmp/*.cubin > $out && rm -rf $tmp && ls -la $out
