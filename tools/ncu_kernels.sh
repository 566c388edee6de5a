# tools/ncu_kernels.sh -- one `ncu --set full` capture per big kernel of the aggregate-verify step (run on the GPU box); the reports
# are turned into the two CSV pages tools/ncu_summary.py reads (the .ncu-rep files themselves exceed gpurun's 64 MiB return limit):
#   gpurun -- 'bash tools/ncu_kernels.sh [name ...]'   then here:  python tools/ncu_summary.py gpurun_out/r2_<k>_raw.csv gpurun_out/r2_<k>_src.csv "<title>"
cap() {  # name regex rounds
  name=$1; rx=$2; rounds=$3
  if [ -n "$ONLY" ] && ! echo " $ONLY " | grep -q " $name "; then return; fi
  timeout 500 ncu --set full --import-source on --clock-control none -k regex:$rx -c 1 -o /tmp/r2_$name python tools/profile_target.py $rounds 1 > gpurun_out/r2_ncu_$name.log 2>&1
  ncu -i /tmp/r2_$name.ncu-rep --page raw --csv > gpurun_out/r2_${name}_raw.csv 2>/dev/null
  ncu -i /tmp/r2_$name.ncu-rep --page source --csv > gpurun_out/r2_${name}_src.csv 2>/dev/null
  rm -f /tmp/r2_$name.ncu-rep
}
ONLY="$*"
cap k_rlc_accum_split 'k_rlc_accum_split' 270336
cap k_rlc_lines_split 'k_rlc_lines_split' 270336
cap k_hash_sw '^k_hash_sw$' 270336
cap k_hash_cofactor_pair '^k_hash_cofactor_pair$' 270336
cap k_g2_decode '^k_g2_decode$' 270336
cap k_g2_subgroup_pair '^k_g2_subgroup_pair$' 270336
cap k_rlc_scale_g1 '^k_rlc_scale_g1$' 270336
cap k_rlc_scale_g2_pair '^k_rlc_scale_g2_pair$' 270336
cap k_mask_aggregate_serial 'k_mask_aggregate_serial' 270336
# latency path: ONE round (a warp per kernel)
export HBLS_HM_CACHE=0
cap k_pairing_coop2 'k_pairing_coop2' 1
cap k_hash_to_g2_coop 'k_hash_to_g2_coop' 1
cap k_g2_decode_pair 'k_g2_decode_pair' 1
