#!/bin/bash
# Text summary of an .ncu-rep for committing under profiles/ (run where ncu is installed; no GPU needed):
#   profiles/summarize.sh prof.ncu-rep > prof_summary.txt
rep="$1"
here="$(cd "$(dirname "$0")" && pwd)"
echo "# $(basename "$rep"): headline metrics (ncu --set full --clock-control none; one replayed launch, cold caches)"
python "$here/ncu_metrics.py" "$rep" l1tex__data_pipe_lsu_wavefronts 2>/dev/null
src="$(mktemp)"; trap 'rm -f "$src"' EXIT
if ncu -i "$rep" --page source --csv > "$src" 2>/dev/null && [ "$(wc -l < "$src")" -gt 10 ] && [ "$(python "$here/ncu_metrics.py" "$rep" 2>/dev/null | head -1 | tr -cd ',' | wc -c)" -eq 0 ]; then
  echo
  echo "# per-instruction view (SASS, --import-source): opcode histogram, shared-memory wavefronts, stall samples"
  python "$here/ncu_source.py" "$src" 30
fi
