// selective-scan forward, warp-private pipeline with two channels per lane, I/O dtype __half (own TU)
#include "scan_fwd_wp2.cuh"
namespace zg {
int scan_fwd_wp2_f16(const zg_scan_params &p, cudaStream_t stream) { return wp2_launch_variant<__half>(p, stream); }
}  // namespace zg
