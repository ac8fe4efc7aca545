// The one reduction every deterministic backward ends with: out[i] += sum_r part[r * n + i], the rows added in row
// order by one thread per column, so the bits of the result are a function of the partials alone (zg_common.cuh).
#include "zg_common.cuh"

namespace zg {

__global__ void __launch_bounds__(256) reduce_rows_kernel(const float *__restrict__ part, int64_t rows, int64_t n, float *__restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float acc = 0.f;
        for (int64_t r = 0; r < rows; ++r) acc += part[r * n + i];
        out[i] += acc;
    }
}

}  // namespace zg

int zg_reduce_rows(const float *part, int64_t rows, int64_t n, float *out, cudaStream_t s) {
    if (rows <= 0 || n <= 0) return 0;
    const int64_t want = (n + 255) / 256;
    const unsigned grid = (unsigned)(want < 132 * 16 ? want : 132 * 16);
    zg::reduce_rows_kernel<<<grid, 256, 0, s>>>(part, rows, n, out);
    zg_count_launch();
    return zg_check_launch("reduce_rows");
}
