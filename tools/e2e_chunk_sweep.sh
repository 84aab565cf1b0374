#!/bin/bash
# End-to-end throughput of the default workload against the pipeline chunk size of the zero-copy path.
#   tools/e2e_chunk_sweep.sh <outdir>
out=${1:?usage: tools/e2e_chunk_sweep.sh <outdir>}
mkdir -p "$out"
for lg in ${LGS:-16 17 18 19}; do
    BNG_ZC_CHUNK_LOG2=$lg timeout -s KILL 100 python bench.py --steps 3 --no-cpu --no-extra --e2e-steps 8 2> "$out/chunk_$lg.err" |
        python -c "import sys,json; j=json.loads(sys.stdin.readline()); print('chunk 2^$lg: e2e', j['e2e']['value'], 'header-split', (j.get('e2e_header_split') or {}).get('value'))"
done | tee "$out/e2e_chunk_sweep.txt"
