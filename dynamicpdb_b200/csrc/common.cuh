// Shared helpers for the dfold_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

namespace dfold {

// last-error buffer shared by every C-ABI entry point (defined in simt.cu)
void set_error(const char* fmt, ...);
int check_launch(const char* what);

#define DFOLD_REQUIRE(cond, ...)                         \
    do {                                                 \
        if (!(cond)) {                                   \
            ::dfold::set_error(__VA_ARGS__);             \
            return 1;                                    \
        }                                                \
    } while (0)

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

static inline long cdiv(long a, long b) { return (a + b - 1) / b; }

// cudaFuncSetAttribute applies to the CURRENT device only (the reference trainer may put the model on any GPU of the
// node): remember, per kernel, what has been configured on each device.
struct SmemCfg { size_t bytes[64] = {}; };
template <typename Kern>
static inline int ensure_dyn_smem(Kern k, size_t bytes, SmemCfg& cfg, const char* name) {
    if (bytes <= 48 * 1024) return 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
    dev &= 63;
    if (cfg.bytes[dev] >= bytes) return 0;
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    DFOLD_REQUIRE(e == cudaSuccess, "%s: cannot reserve %zu B of dynamic shared memory: %s", name, bytes, cudaGetErrorString(e));
    cfg.bytes[dev] = bytes;
    return 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// (w,x,y,z) -> row-major 3x3, un-normalised (|q|^2 R for non-unit q), as openfold rigid_utils.quat_to_rot
__device__ __forceinline__ void quat_to_rot9(float w, float x, float y, float z, float* R) {
    const float ww = w * w, xx = x * x, yy = y * y, zz = z * z;
    const float wx = w * x, wy = w * y, wz = w * z, xy = x * y, xz = x * z, yz = y * z;
    R[0] = ww + xx - yy - zz; R[1] = 2.f * (xy - wz);    R[2] = 2.f * (xz + wy);
    R[3] = 2.f * (xy + wz);   R[4] = ww - xx + yy - zz;  R[5] = 2.f * (yz - wx);
    R[6] = 2.f * (xz - wy);   R[7] = 2.f * (yz + wx);    R[8] = ww - xx - yy + zz;
}

// gradient of quat_to_rot9: given dR[9] accumulate d(w,x,y,z)
__device__ __forceinline__ void quat_to_rot9_bwd(float w, float x, float y, float z, const float* dR,
                                                 float& dw, float& dx, float& dy, float& dz) {
    // R0 = ww+xx-yy-zz ; R4 = ww-xx+yy-zz ; R8 = ww-xx-yy+zz
    dw = 2.f * w * (dR[0] + dR[4] + dR[8]) + 2.f * (-z * dR[1] + y * dR[2] + z * dR[3] - x * dR[5] - y * dR[6] + x * dR[7]);
    dx = 2.f * x * (dR[0] - dR[4] - dR[8]) + 2.f * (y * dR[1] + z * dR[2] + y * dR[3] - w * dR[5] + z * dR[6] + w * dR[7]);
    dy = 2.f * y * (-dR[0] + dR[4] - dR[8]) + 2.f * (x * dR[1] + w * dR[2] + x * dR[3] + z * dR[5] - w * dR[6] + z * dR[7]);
    dz = 2.f * z * (-dR[0] - dR[4] + dR[8]) + 2.f * (-w * dR[1] + x * dR[2] + w * dR[3] + y * dR[5] + x * dR[6] + y * dR[7]);
}

}  // namespace dfold
