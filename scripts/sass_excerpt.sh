#!/bin/bash
# SASS evidence for the instruction claims of DESIGN.md (TMA, mbarrier, packed 16-bit ACS ...), from the objects the product is linked from:
# per hot kernel the register count, the instruction mix of the whole kernel and a few representative lines of every interesting mnemonic.
set -eu
cd "$(dirname "$0")/.."
out=${1:-profiles/sass_excerpts.txt}        # profiles/ is git-ignored: a local record, not source
mkdir -p "$(dirname "$out")"
{
echo "# cuobjdump -sass of welle.io_b200/csrc/build/{ofdm,viterbi}.o (sm_90a), $(date -u +%Y-%m-%d)"
for spec in "ofdm.o|ofdm_demod_kernelILb1ELb0ELb0|UBLKCP SYNCS FMUL FADD MUFU F2I STS.U16 LDS.128" "ofdm.o|find_index_kernelILb1EE|FMUL FADD DSETP DFMA" "viterbi.o|viterbi_kernelILb0|VIMNMX PRMT LDGSTS IDP IMAD.IADD IADD3 STG.E.64 CCTL" "rs.o|superframe_kernel|LDS STS"; do
    obj=${spec%%|*}; rest=${spec#*|}; pat=${rest%%|*}; mn=${rest#*|}
    sass=$(cuobjdump -sass welle.io_b200/csrc/build/$obj | awk -v p="$pat" '$0 ~ "Function : " {f = ($0 ~ p)} f')
    [ -z "$sass" ] && continue
    echo; echo "== $obj :: $(echo "$sass" | head -1 | sed 's/.*Function : //')"
    grep -A3 "$pat" welle.io_b200/csrc/build/${obj%.o}.ptxas.log | grep -E "Used|spill" | head -2 | sed 's/^/   /'
    echo "   instruction mix: $(echo "$sass" | grep -oE '^\s+/\*[0-9a-f]+\*/\s+(@!?U?P[0-9T] )?[A-Z0-9_.]+' | awk '{print $NF}' | sed 's/\..*//' | sort | uniq -c | sort -rn | head -14 | awk '{printf "%s x%s, ", $2, $1}')"
    for m in $mn; do
        n=$(echo "$sass" | grep -cE "\b${m//./\\.}\b" || true)
        echo "   $m x$n:"; echo "$sass" | grep -E "\b${m//./\\.}\b" | head -2 | sed -E 's#/\* 0x[0-9a-f]+ \*/##; s/^ +/        /'
    done
done
} > "$out"
echo "wrote $out"
