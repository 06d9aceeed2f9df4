#!/usr/bin/env bash
# Filtered SASS of one kernel of bagua_b200/_C.so (static evidence of the instruction mix; no GPU needed).
#   scripts/sass_excerpt.sh <mangled-name-regex> > profiles/sass/<name>.txt
set -euo pipefail
PAT="$1"
FILTER='UTCHMMA|UTCBAR|LDTM|UTMALDG|UBLKCP|UTCATOMSWS|SYNCS|UCGABAR|LDGMC|STG\.E.*SYS|LDG\.E.*SYS|ST\.E.*SYS|MULTIMEM|REDG|ATOMG|STG\.E\.128|LDG\.E\.128|MEMBAR'
cuobjdump -sass bagua_b200/_C.so | awk -v pat="$PAT" '/Function : /{p = ($0 ~ pat)} p' > /tmp/sass_one.txt
NAME=$(grep -m1 "Function : " /tmp/sass_one.txt | sed 's/.*Function : //')
echo "// $NAME"
echo "// filtered SASS (cuobjdump -sass, sm_90a): lines matching $FILTER"
grep -E "$FILTER" /tmp/sass_one.txt | sed -E 's/^\s+//' | cut -c1-150
