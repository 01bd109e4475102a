// On-device scan ingest: the raw point rows of every feed that gets a new scan this step, as the files store them (float32 or
// float64 rows of 3 or more values), moved through up to two affine transforms in float64 and written as float32 xyz into the
// feed's half of the live tracker's (feeds, 2, max_points, 3) ping-pong scan buffer (tracking/multi_tracker.py).  One launch
// for any number of feeds: block row y handles descriptor y, the x blocks stride over its rows.
//
// The arithmetic is the readers' (datasets/*.py): p <- R p + t per transform in float64, the products summed in row order,
// then one rounding to float32.  numpy's matmul may sum in another order, so a coordinate can differ by one float32 ulp.
#include "common.cuh"
#include "../../include/o3d_b200.h"

namespace {

constexpr int SI_THREADS = 256;
constexpr int SI_ROWS_PER_THREAD = 4;
constexpr int SI_MAX_STRIDE = 16;
constexpr int SI_MAX_XF = 2;

__device__ __forceinline__ void apply(const double* __restrict__ m, double& x, double& y, double& z) {
    const double a = fma(m[2], z, fma(m[1], y, m[0] * x)) + m[3];
    const double b = fma(m[6], z, fma(m[5], y, m[4] * x)) + m[7];
    const double c = fma(m[10], z, fma(m[9], y, m[8] * x)) + m[11];
    x = a;
    y = b;
    z = c;
}

__global__ void __launch_bounds__(SI_THREADS)
    scan_ingest_kernel(const o3d_scan_desc_t* __restrict__ desc, const unsigned char* __restrict__ slab, int max_points,
                       float* __restrict__ scans, long long* __restrict__ count) {
    __shared__ o3d_scan_desc_t d;
    if (threadIdx.x == 0) d = desc[blockIdx.y];
    __syncthreads();
    const int rows = d.rows, stride = d.stride, nx = d.n_xf;
    const size_t dst = ((size_t)d.feed * 2 + d.half) * (size_t)max_points;
    if (blockIdx.x == 0 && threadIdx.x == 0) count[(size_t)d.feed * 2 + d.half] = rows;
    float* __restrict__ out = scans + dst * 3;
    for (int r = blockIdx.x * SI_THREADS + threadIdx.x; r < rows; r += gridDim.x * SI_THREADS) {
        double x, y, z;
        if (d.is_f64) {
            const double* p = reinterpret_cast<const double*>(slab + d.offset) + (size_t)r * stride;
            x = p[0]; y = p[1]; z = p[2];
        } else {
            const float* p = reinterpret_cast<const float*>(slab + d.offset) + (size_t)r * stride;
            x = p[0]; y = p[1]; z = p[2];
        }
        for (int k = 0; k < nx; ++k) apply(d.xf[k], x, y, z);
        out[(size_t)r * 3 + 0] = (float)x;
        out[(size_t)r * 3 + 1] = (float)y;
        out[(size_t)r * 3 + 2] = (float)z;
    }
}

}  // namespace

extern "C" int o3d_scan_ingest(const o3d_scan_desc_t* desc_host, const o3d_scan_desc_t* desc, int n_desc, const void* slab,
                               long long slab_bytes, int feeds, int max_points, float* scans, long long* count, void* stream) {
    O3D_REQUIRE(desc_host && desc && scans && count && (slab || slab_bytes == 0), O3D_ERR_ARG, "o3d_scan_ingest: null pointer");
    O3D_REQUIRE(n_desc >= 0 && n_desc <= 65535 && feeds >= 1 && max_points >= 1 && slab_bytes >= 0, O3D_ERR_ARG,
                "o3d_scan_ingest: bad sizes n_desc=%d feeds=%d max_points=%d slab_bytes=%lld", n_desc, feeds, max_points, slab_bytes);
    O3D_REQUIRE(n_desc <= 2 * (long long)feeds, O3D_ERR_ARG, "o3d_scan_ingest: n_desc=%d > 2 * feeds", n_desc);
    int most = 0;
    for (int i = 0; i < n_desc; ++i) {
        const o3d_scan_desc_t& d = desc_host[i];
        O3D_REQUIRE(d.feed >= 0 && d.feed < feeds, O3D_ERR_ARG, "o3d_scan_ingest: descriptor %d: feed %d out of [0, %d)", i, d.feed,
                    feeds);
        O3D_REQUIRE(d.half == 0 || d.half == 1, O3D_ERR_ARG, "o3d_scan_ingest: descriptor %d: half %d is not 0 or 1", i, d.half);
        O3D_REQUIRE(d.stride >= 3 && d.stride <= SI_MAX_STRIDE, O3D_ERR_ARG, "o3d_scan_ingest: descriptor %d: stride %d out of [3, %d]",
                    i, d.stride, SI_MAX_STRIDE);
        O3D_REQUIRE(d.is_f64 == 0 || d.is_f64 == 1, O3D_ERR_ARG, "o3d_scan_ingest: descriptor %d: is_f64 %d", i, d.is_f64);
        O3D_REQUIRE(d.n_xf >= 0 && d.n_xf <= SI_MAX_XF, O3D_ERR_ARG, "o3d_scan_ingest: descriptor %d: n_xf %d out of [0, %d]", i,
                    d.n_xf, SI_MAX_XF);
        O3D_REQUIRE(d.rows >= 0 && d.rows <= max_points, O3D_ERR_ARG, "o3d_scan_ingest: descriptor %d: rows %d out of [0, %d]", i,
                    d.rows, max_points);
        const long long elem = d.is_f64 ? 8 : 4;
        O3D_REQUIRE(d.offset >= 0 && d.offset % elem == 0 && d.offset + (long long)d.rows * d.stride * elem <= slab_bytes, O3D_ERR_ARG,
                    "o3d_scan_ingest: descriptor %d: rows at byte %lld (%d x %d x %lld bytes) outside the slab of %lld bytes", i,
                    d.offset, d.rows, d.stride, elem, slab_bytes);
        for (int j = 0; j < i; ++j)
            O3D_REQUIRE(desc_host[j].feed != d.feed || desc_host[j].half != d.half, O3D_ERR_ARG,
                        "o3d_scan_ingest: descriptors %d and %d both write feed %d half %d", j, i, d.feed, d.half);
        most = d.rows > most ? d.rows : most;
    }
    if (n_desc == 0) return O3D_OK;
    const int per_block = SI_THREADS * SI_ROWS_PER_THREAD;
    const dim3 grid((unsigned)((most + per_block - 1) / per_block > 0 ? (most + per_block - 1) / per_block : 1), (unsigned)n_desc);
    scan_ingest_kernel<<<grid, SI_THREADS, 0, (cudaStream_t)stream>>>(desc, static_cast<const unsigned char*>(slab), max_points,
                                                                      scans, count);
    O3D_CHECK_LAUNCH("o3d_scan_ingest");
    return O3D_OK;
}
