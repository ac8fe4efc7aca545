// The DET instantiations of the selective-scan backward kernels (zg_selective_scan_bwd_det), compiled apart from the
// atomic ones in scan_bwd.cu so that the two large translation units build in parallel.
#include "scan_bwd.cuh"

int zg_scan_bwd_launch_det(const zg_scan_bwd_params &q, cudaStream_t s) { return scan_bwd_dispatch<true>(q, s); }
