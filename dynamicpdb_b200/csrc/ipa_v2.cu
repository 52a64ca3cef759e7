// Invariant point attention, second-generation decomposition for the tensor-core path.
//
// The attention probabilities are materialised ONCE as bf16 hi/lo planes  P[F,H,N,N8]  (same bytes as fp32) and
// every dense contraction over them runs on the wgmma split-bf16 GEMM (csrc/gemm_sm90.cu):
//     forward : O = P V                       (batched K-major GEMM, written straight into the concat buffer)
//     backward: dP = dO V^T, dV = P^T dO, dV_pts = P^T dO_pts, dZ = sum_{f,h} P dO_pair
// The kernels here do the part that is NOT a GEMM and must stay exact fp32 on coordinate differences:
//   ipa_prob_fwd   logits = logit0 - gamma/2 * sum_p |q_p - k_p|^2 + mask, exact row softmax (whole rows live in shared
//                  memory), P planes, aggregated global value points, local-frame transform, norms
//   ipa_pair_fwd   o_pair[f,i,h,:] = sum_j P[f,h,i,j] z[i,j,:]   (z row read once for all heads)
//   ipa_ds         dS = P * (dP + dO_pts.v_pts + dO_pair.z - delta), d(gamma)
//   ipa_pts_grad   dq_pts / dk_pts from dS on coordinate differences (tiled, coalesced both ways)
// Reference: src/model/ipa_pytorch_dynamic.py:402-504 and its autograd.
#include "common.cuh"

namespace dfold {
namespace {

constexpr int TI = 32;      // query rows per CTA
constexpr int TJ = 32;      // keys per tile (= warp width)

struct V2Params {
    const float* logit0; long l_fs;        // [Fl,H,N,N]
    const float* q_pts;                    // [F,N,H,Pq,3]
    const float* kv_pts;                   // [F,N,H,Pq+Pv,3]
    const float* pair; long pair_fs;       // [Fz,N,N,Cp]
    const float* quat; const float* trans; // [F,N,4], [F,N,3]
    const float* mask;                     // [F,N]
    const float* gamma;                    // [H]
    uint16_t* p_hi; uint16_t* p_lo; long ldp;   // [F,H,N,ldp]
    float* cat;                            // [F,N,D]
    int F, N, H, C, Pq, Pv, Cp, dfold;
    float inf, eps;
};

__device__ __forceinline__ int cat_width(const V2Params& p) { return p.H * (p.C + (p.dfold ? 8 : 4) * p.Pv + p.Cp); }

__device__ __forceinline__ void split_bf16(float x, uint16_t& hi, uint16_t& lo) {
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
    hi = __bfloat16_as_ushort(h); lo = __bfloat16_as_ushort(l);
}
__device__ __forceinline__ float join_bf16(uint16_t hi, uint16_t lo) {
    return __bfloat162float(__ushort_as_bfloat16(hi)) + __bfloat162float(__ushort_as_bfloat16(lo));
}

// grid (ceil(N/32), H, F), 256 threads; dynamic smem: rows[32][N+1] + q[32][PQ3] + k[32][PQ3+1] + opt[32][PV3]
__global__ void __launch_bounds__(256) ipa_prob_fwd_kernel(const V2Params p) {
    extern __shared__ float sm[];
    const int N = p.N, H = p.H;
    const int PQ3 = p.Pq * 3, PV3 = p.Pv * 3, W = PQ3 + PV3;
    const int LD = N + 1;
    float* s_rows = sm;                         // [TI][LD]
    float* s_q = s_rows + TI * LD;              // [TI][PQ3]
    float* s_k = s_q + TI * PQ3;                // [TJ][PQ3+1]
    float* s_opt = s_k + TJ * (PQ3 + 1);        // [TI][PV3]
    float* s_v = s_opt + TI * PV3;              // [64][PV3]  value-point tile
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int i0 = blockIdx.x * TI, h = blockIdx.y, f = blockIdx.z;

    for (int e = tid; e < TI * PQ3; e += 256) {
        const int r = e / PQ3, c = e % PQ3, i = i0 + r;
        s_q[e] = (i < N) ? p.q_pts[(((long)f * N + i) * H + h) * PQ3 + c] : 0.f;
    }
    const float gam = -0.5f * p.gamma[h];
    const float* l0 = p.logit0 + (long)f * p.l_fs + (long)h * N * N;
    const float* kvp = p.kv_pts + ((long)f * N * H + h) * W;        // + j*H*W
    const float* mrow = p.mask + (long)f * N;

    // ---- phase 1: logits, 4 rows per warp, keys across lanes ----
    for (int j0 = 0; j0 < N; j0 += TJ) {
        __syncthreads();
        for (int e = tid; e < TJ * PQ3; e += 256) {
            const int jj = e / PQ3, c = e % PQ3, j = j0 + jj;
            s_k[jj * (PQ3 + 1) + c] = (j < N) ? kvp[(long)j * H * W + c] : 0.f;
        }
        __syncthreads();
        const int j = j0 + lane;
        if (j < N) {
            const float* kp = s_k + lane * (PQ3 + 1);
            const float mj = mrow[j];
#pragma unroll
            for (int rr = 0; rr < 4; ++rr) {
                const int r = warp * 4 + rr, i = i0 + r;
                float s = 0.f;
                if (i < N) {
                    const float* qp = s_q + r * PQ3;
                    float d2 = 0.f;
                    for (int c = 0; c < PQ3; ++c) { const float d = qp[c] - kp[c]; d2 = fmaf(d, d, d2); }
                    s = l0[(long)i * N + j] + gam * d2 + p.inf * (mrow[i] * mj - 1.f);
                }
                s_rows[r * LD + j] = s;
            }
        }
    }
    __syncthreads();
    // ---- phase 2: exact softmax per row; write P planes ----
#pragma unroll 1
    for (int rr = 0; rr < 4; ++rr) {
        const int r = warp * 4 + rr, i = i0 + r;
        float* row = s_rows + r * LD;
        float m = -INFINITY;
        for (int j = lane; j < N; j += 32) m = fmaxf(m, row[j]);
        m = warp_max(m);
        float sum = 0.f;
        for (int j = lane; j < N; j += 32) { const float e = expf(row[j] - m); row[j] = e; sum += e; }
        sum = warp_sum(sum);
        const float inv = 1.f / sum;
        if (i < N) {
            uint16_t* ph = p.p_hi + (((long)f * H + h) * N + i) * p.ldp;
            uint16_t* pl = p.p_lo + (((long)f * H + h) * N + i) * p.ldp;
            for (int j = lane; j < N; j += 32) {
                const float pv = row[j] * inv;
                row[j] = pv;
                uint16_t a, b;
                split_bf16(pv, a, b);
                ph[j] = a; pl[j] = b;
            }
        }
    }
    __syncthreads();
    // ---- phase 3: aggregated global value points  o_pt[r][e] = sum_j P[r][j] v_pts[j][e]  (key tiles of 64 in smem) ----
    {
        const int r = tid >> 3, g = tid & 7;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};     // comps g, g+8, ... (PV3 <= 64)
        const float* row = s_rows + r * LD;
        const float* vp = kvp + PQ3;
        for (int j0 = 0; j0 < N; j0 += 64) {
            __syncthreads();
            for (int e = tid; e < 64 * PV3; e += 256) {
                const int jj = e / PV3, c = e % PV3, j = j0 + jj;
                s_v[e] = (j < N) ? vp[(long)j * H * W + c] : 0.f;
            }
            __syncthreads();
            const int jn = min(64, N - j0);
            for (int jj = 0; jj < jn; ++jj) {
                const float pv = row[j0 + jj];
                const float* v = s_v + jj * PV3;
#pragma unroll
                for (int m = 0; m < 8; ++m) {
                    const int e = g + 8 * m;
                    if (e < PV3) acc[m] = fmaf(pv, v[e], acc[m]);
                }
            }
        }
#pragma unroll
        for (int m = 0; m < 8; ++m) {
            const int e = g + 8 * m;
            if (e < PV3) s_opt[r * PV3 + e] = acc[m];
        }
    }
    __syncthreads();
    // ---- phase 4: local-frame transform, norms, concat layout ----
    const int D = cat_width(p);
    const int HPv = H * p.Pv;
    const int offLoc = H * p.C, offNl = offLoc + 3 * HPv, offPair = offNl + HPv, offG = offPair + H * p.Cp, offNg = offG + 3 * HPv;
    for (int e = tid; e < TI * p.Pv; e += 256) {
        const int r = e / p.Pv, pt = e % p.Pv, i = i0 + r;
        if (i >= N) continue;
        const float gx = s_opt[r * PV3 + pt * 3], gy = s_opt[r * PV3 + pt * 3 + 1], gz = s_opt[r * PV3 + pt * 3 + 2];
        const long fr = (long)f * N + i;
        const float4 q = *reinterpret_cast<const float4*>(p.quat + 4 * fr);
        float R[9];
        quat_to_rot9(q.x, q.y, q.z, q.w, R);
        const float x = gx - p.trans[3 * fr], y = gy - p.trans[3 * fr + 1], z = gz - p.trans[3 * fr + 2];
        const float lx = R[0] * x + R[3] * y + R[6] * z;
        const float ly = R[1] * x + R[4] * y + R[7] * z;
        const float lz = R[2] * x + R[5] * y + R[8] * z;
        float* orow = p.cat + fr * D;
        const int k = h * p.Pv + pt;
        orow[offLoc + k] = lx; orow[offLoc + HPv + k] = ly; orow[offLoc + 2 * HPv + k] = lz;
        orow[offNl + k] = sqrtf(lx * lx + ly * ly + lz * lz + p.eps);
        if (p.dfold) {
            orow[offG + k] = gx; orow[offG + HPv + k] = gy; orow[offG + 2 * HPv + k] = gz;
            orow[offNg + k] = sqrtf(gx * gx + gy * gy + gz * gz + p.eps);
        }
    }
}

// o_pair[f,i,h,c] = sum_j P[f,h,i,j] z[i,j,c].  grid (N, ceil(F/FG)), 256 threads (8 warps).
// smem: p[H][N] and, when it fits (stage_z), the residue's whole pair row z[i][:][:] — read once and reused by the FG
// frames and all heads of the CTA.
constexpr int FG = 8;
__global__ void __launch_bounds__(256) ipa_pair_fwd_kernel(const V2Params p, int stage_z) {
    extern __shared__ float sm[];
    const int N = p.N, H = p.H, Cp = p.Cp;
    const int i = blockIdx.x;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float* s_p = sm;                          // [H][N]
    float* s_z = sm + H * N;                  // [N][Cp]  (stage_z)
    const int D = cat_width(p);
    const int offPair = H * p.C + 4 * H * p.Pv;
    const bool shared_z = (p.pair_fs == 0);
    if (stage_z && shared_z) {
        const float4* src = reinterpret_cast<const float4*>(p.pair + (long)i * N * Cp);
        float4* dst = reinterpret_cast<float4*>(s_z);
        for (int e = tid; e < N * Cp / 4; e += 256) dst[e] = __ldg(src + e);
    }
    for (int f = blockIdx.y * FG; f < min(p.F, (int)(blockIdx.y + 1) * FG); ++f) {
        __syncthreads();
        for (int e = tid; e < H * N; e += 256) {
            const int h = e / N, j = e % N;
            const long o = (((long)f * H + h) * N + i) * p.ldp + j;
            s_p[e] = join_bf16(p.p_hi[o], p.p_lo[o]);
        }
        if (stage_z && !shared_z) {
            const float4* src = reinterpret_cast<const float4*>(p.pair + (long)f * p.pair_fs + (long)i * N * Cp);
            float4* dst = reinterpret_cast<float4*>(s_z);
            for (int e = tid; e < N * Cp / 4; e += 256) dst[e] = __ldg(src + e);
        }
        __syncthreads();
        const float* zg = p.pair + (long)f * p.pair_fs + (long)i * N * Cp;
        float* orow = p.cat + ((long)f * N + i) * D + offPair;
        for (int h = warp; h < H; h += 8) {
            const float* ph = s_p + h * N;
            for (int c0 = 0; c0 < Cp; c0 += 32) {
                const int c = c0 + lane;
                if (c >= Cp) continue;
                float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
                int j = 0;
                if (stage_z) {
                    for (; j + 4 <= N; j += 4) {
                        a0 = fmaf(ph[j], s_z[j * Cp + c], a0); a1 = fmaf(ph[j + 1], s_z[(j + 1) * Cp + c], a1);
                        a2 = fmaf(ph[j + 2], s_z[(j + 2) * Cp + c], a2); a3 = fmaf(ph[j + 3], s_z[(j + 3) * Cp + c], a3);
                    }
                    for (; j < N; ++j) a0 = fmaf(ph[j], s_z[j * Cp + c], a0);
                } else {
                    for (; j + 4 <= N; j += 4) {
                        const float z0 = __ldg(zg + (long)j * Cp + c), z1 = __ldg(zg + (long)(j + 1) * Cp + c);
                        const float z2 = __ldg(zg + (long)(j + 2) * Cp + c), z3 = __ldg(zg + (long)(j + 3) * Cp + c);
                        a0 = fmaf(ph[j], z0, a0); a1 = fmaf(ph[j + 1], z1, a1);
                        a2 = fmaf(ph[j + 2], z2, a2); a3 = fmaf(ph[j + 3], z3, a3);
                    }
                    for (; j < N; ++j) a0 = fmaf(ph[j], __ldg(zg + (long)j * Cp + c), a0);
                }
                orow[h * Cp + c] = (a0 + a1) + (a2 + a3);
            }
        }
    }
}

// dS[f,h,i,j] = P * (dP + d_og_i . vp_j + dOpair_i . z_ij - delta_i);  dgamma[h] += sum dS * (-0.5 D_ij)
// grid (ceil(N/32), H, F), 256 threads: 4 rows per warp, keys across lanes.
__global__ void __launch_bounds__(256) ipa_ds_kernel(const V2Params p, const float* __restrict__ dcat, const float* __restrict__ d_og,
                                                     const float* __restrict__ delta, const float* __restrict__ dPg,
                                                     const float* __restrict__ Tz,
                                                     float* __restrict__ dS, float* __restrict__ dgamma) {
    extern __shared__ float sm[];
    const int N = p.N, H = p.H, Cp = p.Cp;
    const int PQ3 = p.Pq * 3, PV3 = p.Pv * 3, W = PQ3 + PV3;
    float* s_q = sm;                                 // [TI][PQ3]
    float* s_k = s_q + TI * PQ3;                     // [TJ][W+1]   key points then value points
    float* s_dog = s_k + TJ * (W + 1);               // [TI][PV3]
    float* s_dop = s_dog + TI * PV3;                 // [TI][Cp]
    __shared__ float s_red[8];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int i0 = blockIdx.x * TI, h = blockIdx.y, f = blockIdx.z;
    const int D = cat_width(p);
    const int offPair = H * p.C + 4 * H * p.Pv;
    for (int e = tid; e < TI * PQ3; e += 256) {
        const int r = e / PQ3, c = e % PQ3, i = i0 + r;
        s_q[e] = (i < N) ? p.q_pts[(((long)f * N + i) * H + h) * PQ3 + c] : 0.f;
    }
    for (int e = tid; e < TI * PV3; e += 256) {
        const int r = e / PV3, c = e % PV3, i = i0 + r;
        s_dog[e] = (i < N) ? d_og[(((long)f * N + i) * H + h) * PV3 + c] : 0.f;
    }
    for (int e = tid; e < TI * Cp; e += 256) {
        const int r = e / Cp, c = e % Cp, i = i0 + r;
        s_dop[e] = (i < N) ? dcat[((long)f * N + i) * D + offPair + h * Cp + c] : 0.f;
    }
    const float gam = p.gamma[h];
    const float* kvp = p.kv_pts + ((long)f * N * H + h) * W;
    const float* zbase = p.pair + (long)f * p.pair_fs;
    float dl[4];
#pragma unroll
    for (int rr = 0; rr < 4; ++rr) {
        const int i = i0 + warp * 4 + rr;
        dl[rr] = (i < N) ? delta[((long)f * H + h) * N + i] : 0.f;
    }
    float dgam = 0.f;
    for (int j0 = 0; j0 < N; j0 += TJ) {
        __syncthreads();
        for (int e = tid; e < TJ * W; e += 256) {
            const int jj = e / W, c = e % W, j = j0 + jj;
            s_k[jj * (W + 1) + c] = (j < N) ? kvp[(long)j * H * W + c] : 0.f;
        }
        __syncthreads();
        const int j = j0 + lane;
        if (j >= N) continue;
        const float* kp = s_k + lane * (W + 1);
#pragma unroll
        for (int rr = 0; rr < 4; ++rr) {
            const int r = warp * 4 + rr, i = i0 + r;
            if (i >= N) continue;
            const long o = (((long)f * H + h) * N + i) * N + j;
            const long op = (((long)f * H + h) * N + i) * p.ldp + j;
            const float pv = join_bf16(p.p_hi[op], p.p_lo[op]);
            float dp = dPg[o];
            const float* dg = s_dog + r * PV3;
            for (int c = 0; c < PV3; ++c) dp = fmaf(dg[c], kp[PQ3 + c], dp);
            if (Tz) {
                dp += Tz[((long)i * p.F * H + (long)f * H + h) * N + j];      // sum_c dOpair[f,i,h,c] z[i,j,c]
            } else {
                const float* zr = zbase + ((long)i * N + j) * Cp;
                const float* dz = s_dop + r * Cp;
                for (int c = 0; c < Cp; c += 4) {
                    const float4 z = __ldg(reinterpret_cast<const float4*>(zr + c));
                    dp = fmaf(dz[c], z.x, dp); dp = fmaf(dz[c + 1], z.y, dp);
                    dp = fmaf(dz[c + 2], z.z, dp); dp = fmaf(dz[c + 3], z.w, dp);
                }
            }
            const float ds = pv * (dp - dl[rr]);
            dS[o] = ds;
            const float* qp = s_q + r * PQ3;
            float d2 = 0.f;
            for (int c = 0; c < PQ3; ++c) { const float d = qp[c] - kp[c]; d2 = fmaf(d, d, d2); }
            dgam = fmaf(ds, -0.5f * d2, dgam);
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
    (void)gam;
}

// Second-generation dS kernel (Pq = 8): the value-point term d_og.v_pts arrives precomputed from the tensor cores (Tog,
// [F,H,N,N]), each lane keeps its key's 24 coordinates in registers, the query points are broadcast 16 bytes at a time and
// the squared distance for d(gamma) runs on coordinate pairs held as 64-bit words -- 6 shared-memory loads per pair
// instead of ~120.  sm_90 has no packed FP32 arithmetic: each pair op is two scalar round-to-nearest ops.
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

// transpose = 0: dq_pts[f,a=i,h,c] = -gamma * sum_j dS[i][j] (qp_i - kp_j)
// transpose = 1: dk_pts[f,a=j,h,c] = +gamma * sum_i dS[i][j] (qp_i - kp_j)
// grid (ceil(N/32), H, F), 256 threads: thread = (self item a = tid/8, component group g = tid%8)
__global__ void __launch_bounds__(256) ipa_pts_grad_kernel(const V2Params p, const float* __restrict__ dS, float* __restrict__ dq_pts,
                                                           float* __restrict__ dkv_pts, int transpose) {
    __shared__ float s_w[TI][TJ + 1];
    extern __shared__ float sm[];
    const int N = p.N, H = p.H;
    const int PQ3 = p.Pq * 3, PV3 = p.Pv * 3, W = PQ3 + PV3;
    float* s_self = sm;                     // [32][PQ3]
    float* s_oth = s_self + 32 * PQ3;       // [32][PQ3+1]
    const int tid = threadIdx.x;
    const int a0 = blockIdx.x * 32, h = blockIdx.y, f = blockIdx.z;
    const float* qbase = p.q_pts + ((long)f * N * H + h) * PQ3;     // + i*H*PQ3
    const float* kbase = p.kv_pts + ((long)f * N * H + h) * W;      // + j*H*W
    for (int e = tid; e < 32 * PQ3; e += 256) {
        const int r = e / PQ3, c = e % PQ3, a = a0 + r;
        s_self[e] = (a < N) ? (transpose ? kbase[(long)a * H * W + c] : qbase[(long)a * H * PQ3 + c]) : 0.f;
    }
    const int al = tid >> 3, g = tid & 7;
    float acc[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};                  // comps g + 8m, PQ3 <= 48
    const float* ds = dS + ((long)f * H + h) * N * N;
    for (int b0 = 0; b0 < N; b0 += 32) {
        __syncthreads();
        // dS tile: rows = i, cols = j, coalesced along j
        for (int e = tid; e < 32 * 32; e += 256) {
            const int rr = e >> 5, cc = e & 31;
            const int i = (transpose ? b0 : a0) + rr, j = (transpose ? a0 : b0) + cc;
            s_w[rr][cc] = (i < N && j < N) ? ds[(long)i * N + j] : 0.f;
        }
        for (int e = tid; e < 32 * PQ3; e += 256) {
            const int r = e / PQ3, c = e % PQ3, b = b0 + r;
            s_oth[r * (PQ3 + 1) + c] = (b < N) ? (transpose ? qbase[(long)b * H * PQ3 + c] : kbase[(long)b * H * W + c]) : 0.f;
        }
        __syncthreads();
#pragma unroll 4
        for (int bb = 0; bb < 32; ++bb) {
            const float w = transpose ? s_w[bb][al] : s_w[al][bb];
#pragma unroll
            for (int m = 0; m < 6; ++m) {
                const int c = g + 8 * m;
                if (c < PQ3) {
                    const float sv = s_self[al * PQ3 + c], ov = s_oth[bb * (PQ3 + 1) + c];
                    acc[m] = fmaf(w, transpose ? (ov - sv) : (sv - ov), acc[m]);
                }
            }
        }
    }
    const int a = a0 + al;
    if (a < N) {
        const float gam = p.gamma[h];
#pragma unroll
        for (int m = 0; m < 6; ++m) {
            const int c = g + 8 * m;
            if (c < PQ3) {
                if (!transpose) dq_pts[(((long)f * N + a) * H + h) * PQ3 + c] = -gam * acc[m];
                else dkv_pts[(((long)f * N + a) * H + h) * W + c] = gam * acc[m];
            }
        }
    }
}

}  // namespace
}  // namespace dfold

using namespace dfold;

#define V2_ARGS                                                                                                    \
    const float *logit0, long logit0_fstride, const float *q_pts, const float *kv_pts, const float *pair,          \
        long pair_fstride, const float *quat, const float *trans, const float *mask, const float *gamma,           \
        uint16_t *p_hi, uint16_t *p_lo, long ldp, int F, int N, int H, int C, int Pq, int Pv, int Cp, int dfold,   \
        float inf, float eps

static int v2_params(V2Params& p, V2_ARGS) {
    p.logit0 = logit0; p.l_fs = logit0_fstride; p.q_pts = q_pts; p.kv_pts = kv_pts; p.pair = pair; p.pair_fs = pair_fstride;
    p.quat = quat; p.trans = trans; p.mask = mask; p.gamma = gamma; p.p_hi = p_hi; p.p_lo = p_lo; p.ldp = ldp; p.cat = nullptr;
    p.F = F; p.N = N; p.H = H; p.C = C; p.Pq = Pq; p.Pv = Pv; p.Cp = Cp; p.dfold = dfold; p.inf = inf; p.eps = eps;
    DFOLD_REQUIRE(F > 0 && N > 0 && H > 0 && Pq > 0 && Pv > 0, "ipa_v2: empty problem");
    DFOLD_REQUIRE(Pq * 3 <= 48 && Pv * 3 <= 64 && Cp % 4 == 0, "ipa_v2: unsupported point / pair widths (Pq<=16, Pv<=21, Cp%%4==0)");
    DFOLD_REQUIRE(ldp >= N, "ipa_v2: ldp < N");
    return 0;
}

template <typename Kern>
static int set_smem(Kern k, size_t bytes, const char* name) {
    if (bytes > 48 * 1024) {
        DFOLD_REQUIRE(bytes <= 200 * 1024, "%s: %zu bytes of shared memory needed (sequence too long for this path)", name, bytes);
        cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        DFOLD_REQUIRE(e == cudaSuccess, "%s: cudaFuncSetAttribute(%zu): %s", name, bytes, cudaGetErrorString(e));
    }
    return 0;
}

// Writes the probability planes and the point features of the concat buffer (columns of o and o_pair are filled by
// dfold_gemm_bf16x3_batched and dfold_ipa_pair_fwd).
extern "C" int dfold_ipa_prob_fwd(V2_ARGS, float* out_cat, void* stream) {
    V2Params p;
    if (v2_params(p, logit0, logit0_fstride, q_pts, kv_pts, pair, pair_fstride, quat, trans, mask, gamma, p_hi, p_lo, ldp,
                  F, N, H, C, Pq, Pv, Cp, dfold, inf, eps)) return 1;
    p.cat = out_cat;
    const int PQ3 = Pq * 3, PV3 = Pv * 3;
    const size_t smem = sizeof(float) * (size_t)(TI * (N + 1) + TI * PQ3 + TJ * (PQ3 + 1) + TI * PV3 + 64 * PV3);
    if (set_smem(ipa_prob_fwd_kernel, smem, "ipa_prob_fwd")) return 1;
    dim3 grid((unsigned)cdiv(N, TI), (unsigned)H, (unsigned)F);
    ipa_prob_fwd_kernel<<<grid, 256, smem, as_stream(stream)>>>(p);
    return check_launch("ipa_prob_fwd_kernel");
}

extern "C" int dfold_ipa_pair_fwd(V2_ARGS, float* out_cat, void* stream) {
    V2Params p;
    if (v2_params(p, logit0, logit0_fstride, q_pts, kv_pts, pair, pair_fstride, quat, trans, mask, gamma, p_hi, p_lo, ldp,
                  F, N, H, C, Pq, Pv, Cp, dfold, inf, eps)) return 1;
    p.cat = out_cat;
    size_t smem = sizeof(float) * ((size_t)H * N + (size_t)N * Cp);
    int stage_z = 1;
    if (smem > 160 * 1024) { smem = sizeof(float) * (size_t)H * N; stage_z = 0; }
    if (set_smem(ipa_pair_fwd_kernel, smem, "ipa_pair_fwd")) return 1;
    dim3 grid((unsigned)N, (unsigned)cdiv(F, FG));
    ipa_pair_fwd_kernel<<<grid, 256, smem, as_stream(stream)>>>(p, stage_z);
    return check_launch("ipa_pair_fwd_kernel");
}

// dS [F,H,N,N] from the GEMM-produced dP [F,H,N,N]; dgamma [H] pre-zeroed.  Then the two point-gradient passes.
// Tz (nullable): the pair term sum_c dOpair[f,i,h,c] z[i,j,c] precomputed as [N(i)][F*H][N(j)] on the tensor cores.
extern "C" int dfold_ipa_ds_bwd(V2_ARGS, const float* dcat, const float* d_og, const float* delta, const float* dP,
                                const float* Tz, const float* Tog, float* dS, float* dgamma, float* dq_pts, float* dkv_pts, void* stream) {
    V2Params p;
    if (v2_params(p, logit0, logit0_fstride, q_pts, kv_pts, pair, pair_fstride, quat, trans, mask, gamma, p_hi, p_lo, ldp,
                  F, N, H, C, Pq, Pv, Cp, dfold, inf, eps)) return 1;
    const int PQ3 = Pq * 3, PV3 = Pv * 3, W = PQ3 + PV3;
    cudaStream_t st = as_stream(stream);
    const size_t smem = sizeof(float) * (size_t)(TI * PQ3 + TJ * (W + 1) + TI * PV3 + TI * Cp);
    if (set_smem(ipa_ds_kernel, smem, "ipa_ds")) return 1;
    dim3 grid((unsigned)cdiv(N, TI), (unsigned)H, (unsigned)F);
    if (Tog != nullptr) {
        DFOLD_REQUIRE(Pq == 8 && Tz != nullptr, "dfold_ipa_ds_bwd: the precomputed value-point term needs Pq = 8 and Tz");
        ipa_ds2_kernel<<<grid, 256, 0, st>>>(p, delta, dP, Tz, Tog, dS, dgamma);
        if (check_launch("ipa_ds2_kernel")) return 1;
    } else {
        ipa_ds_kernel<<<grid, 256, smem, st>>>(p, dcat, d_og, delta, dP, Tz, dS, dgamma);
        if (check_launch("ipa_ds_kernel")) return 1;
    }
    if (dq_pts == nullptr) return 0;       // the caller computes the point gradients as tensor-core contractions over dS
    const size_t smem2 = sizeof(float) * (size_t)(32 * PQ3 + 32 * (PQ3 + 1));
    ipa_pts_grad_kernel<<<grid, 256, smem2, st>>>(p, dS, dq_pts, dkv_pts, 0);
    ipa_pts_grad_kernel<<<grid, 256, smem2, st>>>(p, dS, dq_pts, dkv_pts, 1);
    return check_launch("ipa_pts_grad_kernel");
}
