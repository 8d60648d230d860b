#!/bin/bash
# Round-2 `ncu --set full` captures of the kernels named in DESIGN.md / VERDICT (run on the GPU box through gpurun, one GPU).
# .ncu-rep files stay on the box (/tmp); the raw pages are exported as CSV into gpurun_out/ncu_r2/ and summarised by
# profiles/summarise_ncu.py into profiles/ncu_full_r2_summary.json.
set -u
OUT=gpurun_out/ncu_r2
mkdir -p $OUT
NCU="ncu --set full --clock-control none --import-source on"
cap() {  # name, kernel regex, extra ncu args..., -- , python args
  local name=$1 regex=$2; shift 2
  local extra=()
  while [ "$1" != "--" ]; do extra+=("$1"); shift; done
  shift
  timeout 400 $NCU -k "regex:$regex" "${extra[@]}" -f -o /tmp/$name python profiles/ncu_frame.py "$@" > $OUT/$name.log 2>&1
  ncu -i /tmp/$name.ncu-rep --page raw --csv > $OUT/${name}_raw.csv 2>> $OUT/$name.log
  echo "$name rc=$? rows=$(wc -l < $OUT/${name}_raw.csv)"
}
# C2: the HBM-bound named ops (every launch of one eager frame)
cap c2_small "k_pillar_vfe_scatter|k_select|k_cells_insert|k_pyramid_fuse|k_sparse_stem|k_fill_idmap" -- --workload c2 --frames 1
# C2: the wgmma conv, first 26 launches (per-agent ResNet + ResNeXt level 0 + start of level 1) and the tail (deblocks, shrink, heads)
cap c2_conv_head "k_conv2d_tc" --launch-count 26 -- --workload c2 --frames 1
cap c2_conv_tail "k_conv2d_tc" --launch-skip 49 --launch-count 8 -- --workload c2 --frames 1
# C3: tensor-core sparse conv, rulebooks, AttFusion, HeightCompression
cap c3_sparse "k_spconv_tc|k_att_fuse|k_sp_to_bev|k_sp_subm_nbr|k_sp_propose|k_sp_gather_gemm" --launch-count 24 -- --workload c3 --frames 1
# C4: Lift-Splat-Shoot pooling chain + ConvNeXt-free camera trunk pieces
cap c4_lss "k_lss_|k_maxpool3s2|DeviceRadixSort" --launch-count 16 -- --workload c4 --frames 1
ls -la $OUT
