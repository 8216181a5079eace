# DFD_DBG switches of the tensor-core GEMM (csrc/gemm_tc.cu): 1 = skip the TMA store, 2 = skip the statistics pass, 8 = read A from L2
for d in 0 1 8 9; do DFD_DBG=$d GT_ONE=1 python tools/gemm_time.py 2>&1 | grep "stats=False"; done
