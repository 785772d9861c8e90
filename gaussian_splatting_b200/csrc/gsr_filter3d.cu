// gsr_filter3d.cu — Mip-Splatting's 3-D filter size: the finest rate at which any training camera samples each
// gaussian (DESIGN.md 3.13).  One launch replaces Mip-Splatting's Python loop over the cameras (about ten N-sized
// kernels and a masked scatter per camera).
//
//   k_filter3d_min   one thread per gaussian; the cameras pass through shared memory in chunks of F3D_CHUNK, each
//                    thread keeps its minimum r = p_z / max(fx, fy) over the cameras that see it in a register and
//                    writes it (or -1: unseen); the largest r of the seen gaussians goes to one atomicMax on the float
//                    bits (r >= 0, so unsigned order is float order: deterministic)
//   k_filter3d_fill  f = sqrt(variance) * (r, or that largest r for unseen gaussians; 0 when none is seen)
#include "gsr_common.cuh"
#include "gsr_math.cuh"

namespace gsr {

constexpr int F3D_THREADS = 256;
constexpr int F3D_CHUNK = 128;  // cameras per shared-memory pass (21 floats each: 10.5 KB)

struct F3dCam {
    float T[12];                  // rows 0..2 of camera_T_world (transform_point reads M[0..11])
    float fx, cx, fy, cy, rf;     // rf = max(fx, fy)
    float ulo, uhi, vlo, vhi;     // -(m W), (1 + m) W, -(m H), (1 + m) H
};

__global__ void __launch_bounds__(F3D_THREADS) k_filter3d_min(int N, const float* __restrict__ xyz, int C,
                                                              const float* __restrict__ Tc,
                                                              const float* __restrict__ Kc,
                                                              const int* __restrict__ Wc, const int* __restrict__ Hc,
                                                              float near_t, float margin, float* __restrict__ r_out,
                                                              unsigned int* __restrict__ r_max_bits) {
    __shared__ F3dCam cams[F3D_CHUNK];
    const int i = blockIdx.x * F3D_THREADS + threadIdx.x;
    float x = 0.f, y = 0.f, z = 0.f;
    if (i < N) { x = xyz[i * 3 + 0]; y = xyz[i * 3 + 1]; z = xyz[i * 3 + 2]; }
    const float m1 = __fadd_rn(1.0f, margin);
    float r = __int_as_float(0x7f800000);
    bool seen = false;
    for (int c0 = 0; c0 < C; c0 += F3D_CHUNK) {
        const int nc = min(F3D_CHUNK, C - c0);
        __syncthreads();  // the previous chunk is no longer read
        for (int c = threadIdx.x; c < nc; c += F3D_THREADS) {
            const float* T = Tc + (size_t)(c0 + c) * 16;
            const float* K = Kc + (size_t)(c0 + c) * 9;
            F3dCam& cam = cams[c];
#pragma unroll
            for (int k = 0; k < 12; ++k) cam.T[k] = T[k];
            cam.fx = K[0]; cam.cx = K[2]; cam.fy = K[4]; cam.cy = K[5];
            cam.rf = fmaxf(cam.fx, cam.fy);
            const float w = (float)Wc[c0 + c], h = (float)Hc[c0 + c];
            cam.ulo = -__fmul_rn(margin, w); cam.uhi = __fmul_rn(m1, w);
            cam.vlo = -__fmul_rn(margin, h); cam.vhi = __fmul_rn(m1, h);
        }
        __syncthreads();
        if (i < N) {
            for (int c = 0; c < nc; ++c) {  // every thread reads the same camera: shared-memory broadcasts
                const F3dCam& cam = cams[c];
                float px, py, pz, u, v;
                transform_point<float>(cam.T, x, y, z, px, py, pz);
                project_uv<float>(px, py, pz, cam.fx, cam.cx, cam.fy, cam.cy, u, v);
                const bool in = (pz > near_t) & (u >= cam.ulo) & (u <= cam.uhi) & (v >= cam.vlo) & (v <= cam.vhi);
                if (in) {
                    r = fminf(r, __fdiv_rn(pz, cam.rf));
                    seen = true;
                }
            }
        }
    }
    if (i < N) r_out[i] = seen ? r : -1.0f;
    // the largest r of the warp's seen gaussians; one atomic per warp
    unsigned int b = (i < N && seen) ? __float_as_uint(r) : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) b = max(b, __shfl_xor_sync(0xffffffffu, b, o));
    if ((threadIdx.x & 31) == 0 && b != 0u) atomicMax(r_max_bits, b);
}

__global__ void __launch_bounds__(F3D_THREADS) k_filter3d_fill(int N, float sqrt_var,
                                                               const unsigned int* __restrict__ r_max_bits,
                                                               float* __restrict__ f) {
    const int i = blockIdx.x * F3D_THREADS + threadIdx.x;
    if (i >= N) return;
    const float r = f[i];
    f[i] = __fmul_rn(sqrt_var, r < 0.0f ? __uint_as_float(*r_max_bits) : r);
}

}  // namespace gsr

using namespace gsr;

extern "C" int gsr_filter3d(int N, const float* xyz, int C, const float* camera_T_world, const float* K,
                            const int* width, const int* height, float near, float margin, float variance,
                            float* filter3d, void* stream) {
    if (N < 0 || C < 1 || !(near >= 0.0f) || !(margin >= 0.0f) || !(variance >= 0.0f)) return GSR_ERR_BAD_ARG;
    if (N == 0) return GSR_OK;
    if (xyz == nullptr || camera_T_world == nullptr || K == nullptr || width == nullptr || height == nullptr ||
        filter3d == nullptr)
        return GSR_ERR_BAD_ARG;
    cudaStream_t st = (cudaStream_t)stream;
    // 4 bytes of stream-ordered scratch for the maximum (the ABI takes no workspace)
    unsigned int* r_max = nullptr;
    cudaError_t e = cudaMallocAsync((void**)&r_max, sizeof(unsigned int), st);
    if (e != cudaSuccess) return (int)e;
    cudaMemsetAsync(r_max, 0, sizeof(unsigned int), st);
    const int grid = (N + F3D_THREADS - 1) / F3D_THREADS;
    k_filter3d_min<<<grid, F3D_THREADS, 0, st>>>(N, xyz, C, camera_T_world, K, width, height, near, margin, filter3d,
                                                 r_max);
    k_filter3d_fill<<<grid, F3D_THREADS, 0, st>>>(N, sqrtf(variance), r_max, filter3d);
    e = cudaGetLastError();
    cudaFreeAsync(r_max, st);
    return (int)e;
}
