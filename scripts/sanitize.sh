#!/bin/bash
# compute-sanitizer (memcheck + racecheck) over the shared-atomic encoders, the mbarrier / wgmma pipelines of the network kernels
# and the inflate kernel, at small sizes.  Usage: scripts/sanitize.sh OUT_DIR   (logs and a summary land in OUT_DIR)
set -u
OUT=${1:?usage: scripts/sanitize.sh OUT_DIR}
CS=${CUDA_HOME:-/usr/local/cuda}/bin/compute-sanitizer
mkdir -p "$OUT"
run() {  # name tool pytest-args...
    local name=$1 tool=$2; shift 2
    timeout 900 "$CS" --tool $tool --print-limit 5 --error-exitcode 86 --log-file "$OUT/sanitizer_${name}_${tool}.log" \
        python -m pytest -x -q -p no:cacheprovider "$@" > "$OUT/sanitizer_${name}_${tool}.pytest" 2>&1
    echo "$name $tool exit=$? $(tail -1 "$OUT/sanitizer_${name}_${tool}.pytest")" | tee -a "$OUT/sanitizer_summary.txt"
    tail -3 "$OUT/sanitizer_${name}_${tool}.log" >> "$OUT/sanitizer_summary.txt"
}
: > "$OUT/sanitizer_summary.txt"
for tool in memcheck racecheck; do
    run variant_encoder $tool tests/test_variant_encoder_gpu.py -k "kats or empty_and_small"          # k_tile_count, k_collect_ops, k_site_alleles, k_windows
    run polish_encoder $tool tests/test_polish_encoder_gpu.py -k "kat"                                 # k_polish_count
    run nets_variant $tool "tests/test_nets_gpu.py::test_variant_net_vs_oracle[130-2-1]"                 # k_lstm_layer, k_tc_gemm_p
    run nets_polish $tool "tests/test_nets_gpu.py::test_polish_net_vs_oracle[5-5-1]"                     # k_gru_layer
    run inflate $tool tests/test_inflate_gpu.py tests/test_inflate_edges_gpu.py -k "inflate_matches or rejects or case_table or cut_short"   # k_bgzf_inflate
    run realign $tool tests/test_realign_edges_gpu.py -k "reject or (match_port and 8)"                # k_sw16<8>, k_banded
    run stitch_sink $tool tests/test_polish_assembly_gpu.py -k "stitch_sink"                           # k_stitch_sink
    run vcf $tool tests/test_genome_vcf_gpu.py -k "vcf_host"                                         # k_site_sizes, k_site_write
    run bgzf_deflate $tool tests/test_genome_dist_gpu.py -k "compressor"                             # k_bgzf_deflate, k_bgzf_compact
    run gvcf $tool tests/test_gvcf_gpu.py -k "block_pass and 1 or track_matches"                    # k_gvcf_*, k_tile_count track store
done
cat "$OUT/sanitizer_summary.txt"
