// Invariant point attention, backward of the tensor-core path (preset-A head geometry, Pq = 8).
//
// The forward (csrc/ipa_fused.cu) materialises the attention probabilities ONCE as bf16 hi/lo planes  P[F,H,N,ldp]  (same
// bytes as fp32), and every dense contraction of the backward runs on the wgmma split-bf16 GEMM (csrc/gemm_sm90.cu):
//     dP = dO V^T, the pair term Tz = dO_pair.z, the value-point term Tog = d_og.v_pts, dV = P^T dO, dV_pts = P^T dO_pts,
//     dZ = sum_{f,h} P dO_pair, and the point gradients dS K_pts, dS^T Q_pts.
// The kernel here is the part that is NOT a GEMM and must stay exact fp32 on coordinate differences:
//   ipa_ds2   dS = P * (dP + Tog + Tz - delta), per-CTA partials of d(gamma) = sum dS * (-1/2 |q_i - k_j|^2)
// Reference: src/model/ipa_pytorch_dynamic.py:402-504 and its autograd.
#include "common.cuh"

namespace dfold {
namespace {

constexpr int TI = 32;      // query rows per CTA
constexpr int TJ = 32;      // keys per tile (= warp width)

struct V2Params {
    const float* q_pts;                                 // [F,N,H,8,3]
    const float* kv_pts;                                // [F,N,H,8+Pv,3]
    const uint16_t* p_hi; const uint16_t* p_lo; long ldp;   // [F,H,N,ldp]
    int F, N, H, Pv;
};

__device__ __forceinline__ float join_bf16(uint16_t hi, uint16_t lo) {
    return __bfloat162float(__ushort_as_bfloat16(hi)) + __bfloat162float(__ushort_as_bfloat16(lo));
}

// dS kernel (Pq = 8): the value-point term d_og.v_pts arrives precomputed from the tensor cores (Tog, [F,H,N,N]), each lane
// keeps its key's 24 coordinates in registers, the query points are broadcast 16 bytes at a time and the squared distance
// for d(gamma) runs on coordinate pairs held as 64-bit words -- 6 shared-memory loads per pair instead of ~120.  sm_90 has
// no packed FP32 arithmetic: each pair op is two scalar round-to-nearest ops.
// grid (ceil(N/32), H, F), 256 threads: 4 rows per warp, keys across lanes.
typedef unsigned long long u64v2;
__device__ __forceinline__ u64v2 v2_sub2(u64v2 a, u64v2 b) {
    const float2 x = *reinterpret_cast<const float2*>(&a), y = *reinterpret_cast<const float2*>(&b);
    const float2 r = make_float2(__fsub_rn(x.x, y.x), __fsub_rn(x.y, y.y));
    return *reinterpret_cast<const u64v2*>(&r);
}
__device__ __forceinline__ u64v2 v2_fma2(u64v2 a, u64v2 b, u64v2 c) {
    const float2 x = *reinterpret_cast<const float2*>(&a), y = *reinterpret_cast<const float2*>(&b), z = *reinterpret_cast<const float2*>(&c);
    const float2 r = make_float2(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
    return *reinterpret_cast<const u64v2*>(&r);
}
__global__ void __launch_bounds__(256) ipa_ds2_kernel(const V2Params p, const float* __restrict__ delta, const float* __restrict__ dPg,
                                                      const float* __restrict__ Tz, const float* __restrict__ Tog,
                                                      float* __restrict__ dS, float* __restrict__ dgamma) {
    __shared__ __align__(16) float s_q[TI * 24];
    __shared__ __align__(16) float s_k[TJ * 24];
    __shared__ float s_red[8];
    const int N = p.N, H = p.H;
    const int W = 24 + p.Pv * 3;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int i0 = blockIdx.x * TI, h = blockIdx.y, f = blockIdx.z;
    for (int e = tid; e < TI * 6; e += 256) {
        const int r = e / 6, c4 = e % 6, i = i0 + r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < N) v = __ldg(reinterpret_cast<const float4*>(p.q_pts + (((long)f * N + i) * H + h) * 24) + c4);
        reinterpret_cast<float4*>(s_q)[e] = v;
    }
    const float* kvp = p.kv_pts + ((long)f * N * H + h) * W;
    float dl[4];
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
        const int i = i0 + warp * 4 + rr;
        dl[rr] = (i < N) ? delta[((long)f * H + h) * N + i] : 0.f;
    }
    float dgam = 0.f;
    for (int j0 = 0; j0 < N; j0 += TJ) {
        __syncthreads();
        for (int e = tid; e < TJ * 6; e += 256) {
            const int jj = e / 6, c4 = e % 6, j = j0 + jj;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (j < N) v = __ldg(reinterpret_cast<const float4*>(kvp + (long)j * H * W) + c4);
            reinterpret_cast<float4*>(s_k)[e] = v;
        }
        __syncthreads();
        const int j = j0 + lane;
        if (j >= N) continue;
        u64v2 k[12];
#pragma unroll
        for (int c = 0; c < 6; ++c) {
            const ulonglong2 v = reinterpret_cast<const ulonglong2*>(s_k + lane * 24)[c];
            k[2 * c] = v.x; k[2 * c + 1] = v.y;
        }
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) {
            const int r = warp * 4 + rr, i = i0 + r;
            if (i >= N) continue;
            const long o = (((long)f * H + h) * N + i) * N + j;
            const long op = (((long)f * H + h) * N + i) * p.ldp + j;
            const float pv = join_bf16(p.p_hi[op], p.p_lo[op]);
            const float dp = dPg[o] + Tog[o] + Tz[((long)i * p.F * H + (long)f * H + h) * N + j];
            const float ds = pv * (dp - dl[rr]);
            dS[o] = ds;
            const ulonglong2* q2 = reinterpret_cast<const ulonglong2*>(s_q + r * 24);
            u64v2 a0 = 0ull;
#pragma unroll
            for (int c = 0; c < 6; ++c) {
                const ulonglong2 qq = q2[c];
                const u64v2 d0 = v2_sub2(qq.x, k[2 * c]), d1 = v2_sub2(qq.y, k[2 * c + 1]);
                a0 = v2_fma2(d0, d0, a0);
                a0 = v2_fma2(d1, d1, a0);
            }
            float x0, x1;
            asm("mov.b64 {%0, %1}, %2;" : "=f"(x0), "=f"(x1) : "l"(a0));
            dgam = fmaf(ds, -0.5f * (x0 + x1), dgam);
        }
    }
    dgam = warp_sum(dgam);
    if (lane == 0) s_red[warp] = dgam;
    __syncthreads();
    if (tid == 0) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += s_red[w];
        dgamma[(long)h * p.F * p.N + (long)blockIdx.z * gridDim.x + blockIdx.x] = t;   // per-CTA partial (no atomics)
    }
}

}  // namespace
}  // namespace dfold

using namespace dfold;

// dS [F,H,N,N] from the GEMM-produced dP [F,H,N,N] and the precomputed pair (Tz) and value-point (Tog) terms; dgamma
// partials [H][F*N] pre-zeroed.
extern "C" int dfold_ipa_ds_bwd(const float* q_pts, const float* kv_pts, const uint16_t* p_hi, const uint16_t* p_lo, long ldp,
                                int F, int N, int H, int Pq, int Pv, const float* delta, const float* dP, const float* Tz,
                                const float* Tog, float* dS, float* dgamma, void* stream) {
    DFOLD_REQUIRE(F > 0 && N > 0 && H > 0 && Pv > 0, "dfold_ipa_ds_bwd: empty problem");
    DFOLD_REQUIRE(Pq == 8, "dfold_ipa_ds_bwd: Pq = %d, the kernel holds 8 query / key points per head", Pq);
    DFOLD_REQUIRE(Pv % 4 == 0, "dfold_ipa_ds_bwd: Pv = %d, key rows of 24 + 3 Pv floats are read as float4", Pv);
    DFOLD_REQUIRE(ldp >= N, "dfold_ipa_ds_bwd: ldp < N");
    DFOLD_REQUIRE(Tz != nullptr && Tog != nullptr, "dfold_ipa_ds_bwd: the pair and value-point terms Tz and Tog are required");
    const V2Params p{q_pts, kv_pts, p_hi, p_lo, ldp, F, N, H, Pv};
    dim3 grid((unsigned)cdiv(N, TI), (unsigned)H, (unsigned)F);
    ipa_ds2_kernel<<<grid, 256, 0, as_stream(stream)>>>(p, delta, dP, Tz, Tog, dS, dgamma);
    return check_launch("ipa_ds2_kernel");
}
