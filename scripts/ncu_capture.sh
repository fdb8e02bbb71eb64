#!/bin/bash
# One `ncu --set full` capture per hot kernel (1 GPU). Reports land in $MIMO_OUT/ncu_*.ncu-rep (default mimo_out/).
OUT=${MIMO_OUT:-mimo_out}
mkdir -p $OUT
SPECS=("$@")
if [ ${#SPECS[@]} -eq 0 ]; then SPECS=("gemm:gemm_wgmma_kernel" "geglu:gemm_wgmma_kernel" "conv:gemm_wgmma_kernel" "attn:attn_spatial_kernel" "attn80:attn_spatial_kernel" "norm:gn_apply_kernel" "norm:layernorm_kernel" "temporal:attn_temporal_kernel"); fi
for spec in "${SPECS[@]}"; do
  fn=${spec%%:*}; kn=${spec##*:}
  out=$OUT/ncu_${fn}_${kn}
  timeout 300 ncu --set full --clock-control none --import-source on -k regex:$kn -s 2 -c 1 -f -o $out \
      python scripts/ncu_kernels.py $fn > $OUT/ncu_${fn}_${kn}.log 2>&1
  echo "$spec exit=$?"
done
ls -la $OUT/*.ncu-rep
