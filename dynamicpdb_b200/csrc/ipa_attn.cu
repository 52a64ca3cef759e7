// Fused invariant-point-attention core for sm_90a.
//
// One kernel does: scalar logits (+pair bias, precomputed by the tensor-core GEMM) + point-distance term on
// coordinate DIFFERENCES + mask + online softmax + value / value-point / pair aggregation + local-frame
// inverse transform + norms, and writes the concat buffer that feeds linear_out.  Nothing of size N x N x H x P
// is ever materialised (the reference materialises [nf,N,N,H,Pq,3] and [nf,H,3,N,N,Pv], SURVEY.md §8 a3).
//
// Replaces src/model/ipa_pytorch_dynamic.py:402-504 (DFOLD fork, dfold=1) and
// openfold/model/structure_module.py:315-428 (vanilla, dfold=0).
//
// Work decomposition: CTA = (query tile of TI residues, head h, frame f).  Threads are a grid of
// (row group rg) x (channel group cg): each thread owns RT rows x 4 channels of the per-head output row
//   [ v (C) | value points (3*Pv) | pair (Cp) ],
// so value rows are read once per key as float4 and reused for RT query rows from registers; the softmax
// statistics use warp shuffles (one warp per query row, 32 keys per tile).
#include "common.cuh"

namespace dfold {
namespace {

constexpr int TJ = 32;      // keys per tile == warp width
constexpr int RT = 8;       // query rows per thread

struct IpaParams {
    const float* logit0; long l_fs;        // [Fl,H,N,N]
    const float* kv; long kv_fs;           // [Fs,N,H,2C]  (per head [K | V])
    const float* q_pts;                    // [F,N,H,Pq,3]
    const float* kv_pts;                   // [F,N,H,Pq+Pv,3]
    const float* pair; long pair_fs;       // [Fz,N,N,Cp]
    const float* quat; const float* trans; // [F,N,4], [F,N,3]
    const float* mask;                     // [F,N]
    const float* gamma;                    // [H]  softplus(w) * sqrt(1/(3*Pq*9/2))
    float* out;                            // [F,N,D]
    float* lse;                            // [F,H,N]
    int F, N, H, C, Pq, Pv, Cp, dfold;
    int C4, P4, Z4, CGP, RG;               // thread-grid geometry
    float inf, eps;
};

__device__ __forceinline__ int concat_width(const IpaParams& p) {
    return p.H * (p.C + (p.dfold ? 8 : 4) * p.Pv + p.Cp);
}

__global__ void ipa_fwd_kernel(const IpaParams p) {
    extern __shared__ float sm[];
    const int TI = p.RG * RT;
    const int PQ3 = p.Pq * 3, PV3 = p.Pv * 3;
    const int SW = max(TJ + 1, PV3);                 // row width of the logits / o_pt scratch
    float* s_q = sm;                                 // [TI][PQ3]
    float* s_k = s_q + TI * PQ3;                     // [TJ][PQ3+1]
    float* s_s = s_k + TJ * (PQ3 + 1);               // [TI][SW]   raw logits of the tile; later o_pt
    float* s_p = s_s + TI * SW;                      // [TJ][TI]   probabilities, key-major
    float* s_m = s_p + TJ * TI;                      // [TI] running max
    float* s_l = s_m + TI;                           // [TI] running sum
    float* s_c = s_l + TI;                           // [TI] rescale factor of this tile

    const int tid = threadIdx.x, nthr = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarp = nthr >> 5;
    const int i0 = blockIdx.x * TI, h = blockIdx.y, f = blockIdx.z;
    const int N = p.N, H = p.H, C = p.C;
    const int cg = tid % p.CGP, rg = tid / p.CGP;
    const int cgTot = p.C4 + p.P4 + p.Z4;
    const int seg = (cg < p.C4) ? 0 : (cg < p.C4 + p.P4 ? 1 : (cg < cgTot ? 2 : 3));

    for (int e = tid; e < TI * PQ3; e += nthr) {
        const int r = e / PQ3, c = e % PQ3;
        const int i = i0 + r;
        s_q[e] = (i < N) ? p.q_pts[(((long)f * N + i) * H + h) * PQ3 + c] : 0.f;
    }
    for (int r = tid; r < TI; r += nthr) { s_m[r] = -INFINITY; s_l[r] = 0.f; }

    float acc[RT][4];
#pragma unroll
    for (int r = 0; r < RT; ++r) { acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f; }

    const float gam = -0.5f * p.gamma[h];
    const float* l0 = p.logit0 + (long)f * p.l_fs + (long)h * N * N;
    const float* vbase = p.kv + (long)f * p.kv_fs + (long)h * 2 * C + C;
    const float* kvp = p.kv_pts + (long)f * N * H * (PQ3 + PV3) + (long)h * (PQ3 + PV3);
    const float* zbase = p.pair + (long)f * p.pair_fs;
    const float* mrow = p.mask + (long)f * N;

    for (int j0 = 0; j0 < N; j0 += TJ) {
        __syncthreads();     // previous tile fully consumed (s_k, s_s, s_p reuse)
        for (int e = tid; e < TJ * PQ3; e += nthr) {
            const int jj = e / PQ3, c = e % PQ3;
            const int j = j0 + jj;
            s_k[jj * (PQ3 + 1) + c] = (j < N) ? kvp[(long)j * H * (PQ3 + PV3) + c] : 0.f;
        }
        __syncthreads();
        // ---- logits of the tile: one (row, key) pair per thread-iteration, keys across lanes ----
        for (int e = tid; e < TI * TJ; e += nthr) {
            const int r = e / TJ, jj = e % TJ;
            const int i = i0 + r, j = j0 + jj;
            float s = -INFINITY;
            if (i < N && j < N) {
                float d2 = 0.f;
                const float* qp = s_q + r * PQ3;
                const float* kp = s_k + jj * (PQ3 + 1);
                for (int c = 0; c < PQ3; ++c) { const float d = qp[c] - kp[c]; d2 = fmaf(d, d, d2); }
                s = l0[(long)i * N + j] + gam * d2 + p.inf * (mrow[i] * mrow[j] - 1.f);
            } else if (j < N) {
                s = 0.f;      // padded query row: keep finite, never written out
            }
            s_s[r * SW + jj] = s;
        }
        __syncthreads();
        // ---- online softmax: warp per row ----
        for (int r = warp; r < TI; r += nwarp) {
            const float s = s_s[r * SW + lane];
            const float m_old = s_m[r];
            const float m_new = fmaxf(m_old, warp_max(s));
            const float pe = expf(s - m_new);
            const float sum = warp_sum(pe);
            s_p[lane * TI + r] = pe;
            if (lane == 0) {
                const float sc = expf(m_old - m_new);
                s_c[r] = sc;
                s_l[r] = s_l[r] * sc + sum;
                s_m[r] = m_new;
            }
        }
        __syncthreads();
        // ---- accumulate ----
        if (seg < 3) {
#pragma unroll
            for (int r = 0; r < RT; ++r) {
                const float sc = s_c[rg * RT + r];
                acc[r][0] *= sc; acc[r][1] *= sc; acc[r][2] *= sc; acc[r][3] *= sc;
            }
            const int jmax = min(TJ, N - j0);
            for (int jj = 0; jj < jmax; ++jj) {
                const int j = j0 + jj;
                float pr[RT];
                const float4* pp = reinterpret_cast<const float4*>(s_p + jj * TI + rg * RT);
                const float4 p0 = pp[0], p1 = pp[1];
                pr[0] = p0.x; pr[1] = p0.y; pr[2] = p0.z; pr[3] = p0.w;
                pr[4] = p1.x; pr[5] = p1.y; pr[6] = p1.z; pr[7] = p1.w;
                if (seg == 0) {
                    const float4 v = __ldg(reinterpret_cast<const float4*>(vbase + (long)j * H * 2 * C + cg * 4));
#pragma unroll
                    for (int r = 0; r < RT; ++r) {
                        acc[r][0] = fmaf(pr[r], v.x, acc[r][0]); acc[r][1] = fmaf(pr[r], v.y, acc[r][1]);
                        acc[r][2] = fmaf(pr[r], v.z, acc[r][2]); acc[r][3] = fmaf(pr[r], v.w, acc[r][3]);
                    }
                } else if (seg == 1) {
                    const int e0 = (cg - p.C4) * 4;
                    const float* vp = kvp + (long)j * H * (PQ3 + PV3) + PQ3 + e0;
                    float v[4];
#pragma unroll
                    for (int c = 0; c < 4; ++c) v[c] = (e0 + c < PV3) ? __ldg(vp + c) : 0.f;
#pragma unroll
                    for (int r = 0; r < RT; ++r) {
                        acc[r][0] = fmaf(pr[r], v[0], acc[r][0]); acc[r][1] = fmaf(pr[r], v[1], acc[r][1]);
                        acc[r][2] = fmaf(pr[r], v[2], acc[r][2]); acc[r][3] = fmaf(pr[r], v[3], acc[r][3]);
                    }
                } else {
                    const int c4 = cg - p.C4 - p.P4;
#pragma unroll
                    for (int r = 0; r < RT; ++r) {
                        const int i = i0 + rg * RT + r;
                        if (i < N) {
                            const float4 z = __ldg(reinterpret_cast<const float4*>(zbase + ((long)i * N + j) * p.Cp + c4 * 4));
                            acc[r][0] = fmaf(pr[r], z.x, acc[r][0]); acc[r][1] = fmaf(pr[r], z.y, acc[r][1]);
                            acc[r][2] = fmaf(pr[r], z.z, acc[r][2]); acc[r][3] = fmaf(pr[r], z.w, acc[r][3]);
                        }
                    }
                }
            }
        }
    }
    __syncthreads();
    // ---- epilogue ----
    const int D = concat_width(p);
    const int HPv = H * p.Pv;
    const int offLoc = H * C, offNl = offLoc + 3 * HPv, offPair = offNl + HPv, offG = offPair + H * p.Cp, offNg = offG + 3 * HPv;
#pragma unroll
    for (int r = 0; r < RT; ++r) {
        const int rr = rg * RT + r;
        const int i = i0 + rr;
        if (i >= N || seg == 3) continue;
        const float inv = 1.f / s_l[rr];
        float* orow = p.out + ((long)f * N + i) * D;
        if (seg == 0) {
            *reinterpret_cast<float4*>(orow + h * C + cg * 4) =
                make_float4(acc[r][0] * inv, acc[r][1] * inv, acc[r][2] * inv, acc[r][3] * inv);
        } else if (seg == 2) {
            const int c4 = cg - p.C4 - p.P4;
            *reinterpret_cast<float4*>(orow + offPair + h * p.Cp + c4 * 4) =
                make_float4(acc[r][0] * inv, acc[r][1] * inv, acc[r][2] * inv, acc[r][3] * inv);
        } else {
            const int e0 = (cg - p.C4) * 4;
#pragma unroll
            for (int c = 0; c < 4; ++c)
                if (e0 + c < PV3) s_s[rr * SW + e0 + c] = acc[r][c] * inv;
        }
    }
    __syncthreads();
    for (int e = tid; e < TI * p.Pv; e += nthr) {
        const int rr = e / p.Pv, pt = e % p.Pv;
        const int i = i0 + rr;
        if (i >= N) continue;
        const float gx = s_s[rr * SW + pt * 3], gy = s_s[rr * SW + pt * 3 + 1], gz = s_s[rr * SW + pt * 3 + 2];
        const long fr = (long)f * N + i;
        const float4 q = *reinterpret_cast<const float4*>(p.quat + 4 * fr);
        float R[9];
        quat_to_rot9(q.x, q.y, q.z, q.w, R);
        const float x = gx - p.trans[3 * fr], y = gy - p.trans[3 * fr + 1], z = gz - p.trans[3 * fr + 2];
        const float lx = R[0] * x + R[3] * y + R[6] * z;
        const float ly = R[1] * x + R[4] * y + R[7] * z;
        const float lz = R[2] * x + R[5] * y + R[8] * z;
        float* orow = p.out + fr * D;
        const int k = h * p.Pv + pt;
        orow[offLoc + k] = lx; orow[offLoc + HPv + k] = ly; orow[offLoc + 2 * HPv + k] = lz;
        orow[offNl + k] = sqrtf(lx * lx + ly * ly + lz * lz + p.eps);
        if (p.dfold) {
            orow[offG + k] = gx; orow[offG + HPv + k] = gy; orow[offG + 2 * HPv + k] = gz;
            orow[offNg + k] = sqrtf(gx * gx + gy * gy + gz * gz + p.eps);
        }
    }
    for (int r = tid; r < TI; r += nthr)
        if (i0 + r < N) p.lse[((long)f * H + h) * N + i0 + r] = s_m[r] + logf(s_l[r]);
}

// ---------------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------------
// B0: per (f, i): undo the local-frame epilogue.  One warp per (f,i); lanes over (h, point).
//   d_og[F,N,H,Pv,3]  total gradient w.r.t. the global-frame aggregated points
//   delta[F,H,N]      sum_c dO * O over every aggregated channel (v, global points, pair)
//   dquat[F,N,4], dtrans[F,N,3]  gradient through  ol = R^T (og - t)
__global__ void ipa_bwd_pre_kernel(const IpaParams p, const float* __restrict__ cat, const float* __restrict__ dcat,
                                   float* __restrict__ d_og, float* __restrict__ delta,
                                   float* __restrict__ dquat, float* __restrict__ dtrans) {
    const long fr = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (fr >= (long)p.F * p.N) return;
    const int lane = threadIdx.x & 31;
    const int H = p.H, C = p.C, Pv = p.Pv, Cp = p.Cp, N = p.N;
    const int f = (int)(fr / N), i = (int)(fr % N);
    const int D = concat_width(p);
    const int HPv = H * Pv;
    const int offLoc = H * C, offNl = offLoc + 3 * HPv, offPair = offNl + HPv, offG = offPair + H * Cp, offNg = offG + 3 * HPv;
    const float* o = cat + fr * D;
    const float* g = dcat + fr * D;
    const float4 q = *reinterpret_cast<const float4*>(p.quat + 4 * fr);
    float R[9];
    quat_to_rot9(q.x, q.y, q.z, q.w, R);
    const float tx = p.trans[3 * fr], ty = p.trans[3 * fr + 1], tz = p.trans[3 * fr + 2];
    float dR[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float dt[3] = {0.f, 0.f, 0.f};
    for (int h = 0; h < H; ++h) {
        float dl = 0.f;
        for (int c = lane; c < C; c += 32) dl = fmaf(g[h * C + c], o[h * C + c], dl);
        for (int c = lane; c < Cp; c += 32) dl = fmaf(g[offPair + h * Cp + c], o[offPair + h * Cp + c], dl);
        for (int pt = lane; pt < Pv; pt += 32) {
            const int k = h * Pv + pt;
            const float lx = o[offLoc + k], ly = o[offLoc + HPv + k], lz = o[offLoc + 2 * HPv + k];
            const float nl = o[offNl + k];
            const float gn = g[offNl + k] / nl;
            // total gradient on the local point
            const float ax = g[offLoc + k] + gn * lx, ay = g[offLoc + HPv + k] + gn * ly, az = g[offLoc + 2 * HPv + k] + gn * lz;
            // global point (saved for dfold; reconstructed otherwise)
            float ogx, ogy, ogz;
            if (p.dfold) { ogx = o[offG + k]; ogy = o[offG + HPv + k]; ogz = o[offG + 2 * HPv + k]; }
            else {
                ogx = R[0] * lx + R[1] * ly + R[2] * lz + tx;
                ogy = R[3] * lx + R[4] * ly + R[5] * lz + ty;
                ogz = R[6] * lx + R[7] * ly + R[8] * lz + tz;
            }
            // ol_b = sum_a R[a][b] (og - t)_a
            float rx = R[0] * ax + R[1] * ay + R[2] * az;
            float ry = R[3] * ax + R[4] * ay + R[5] * az;
            float rz = R[6] * ax + R[7] * ay + R[8] * az;
            dt[0] -= rx; dt[1] -= ry; dt[2] -= rz;
            const float ux = ogx - tx, uy = ogy - ty, uz = ogz - tz;
            dR[0] += ux * ax; dR[1] += ux * ay; dR[2] += ux * az;
            dR[3] += uy * ax; dR[4] += uy * ay; dR[5] += uy * az;
            dR[6] += uz * ax; dR[7] += uz * ay; dR[8] += uz * az;
            if (p.dfold) {
                const float gg = g[offNg + k] / o[offNg + k];
                rx += g[offG + k] + gg * ogx; ry += g[offG + HPv + k] + gg * ogy; rz += g[offG + 2 * HPv + k] + gg * ogz;
            }
            float* dst = d_og + ((fr * H + h) * Pv + pt) * 3;
            dst[0] = rx; dst[1] = ry; dst[2] = rz;
            dl += rx * ogx + ry * ogy + rz * ogz;
        }
        dl = warp_sum(dl);
        if (lane == 0) delta[((long)f * H + h) * N + i] = dl;
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) dR[k] = warp_sum(dR[k]);
#pragma unroll
    for (int k = 0; k < 3; ++k) dt[k] = warp_sum(dt[k]);
    if (lane == 0) {
        float dw, dx, dy, dz;
        quat_to_rot9_bwd(q.x, q.y, q.z, q.w, dR, dw, dx, dy, dz);
        *reinterpret_cast<float4*>(dquat + 4 * fr) = make_float4(dw, dx, dy, dz);
        dtrans[3 * fr] = dt[0]; dtrans[3 * fr + 1] = dt[1]; dtrans[3 * fr + 2] = dt[2];
    }
}

// B1: CTA = (query tile of 32 rows, head, frame), 256 threads: warp w owns rows 4w..4w+3, lanes = 32 keys.
// Recomputes P from lse, forms dP = dO.V^T (+ point and pair terms) and dS = P (dP - delta), writes both
// head-major  P, dS : [H, F, N, N]  and accumulates d(gamma).
constexpr int B1_TI = 32;
constexpr int B1_RB = 4;
__global__ void __launch_bounds__(256) ipa_bwd_row_kernel(const IpaParams p, const float* __restrict__ dcat,
                                                          const float* __restrict__ d_og, const float* __restrict__ delta,
                                                          float* __restrict__ Pm, float* __restrict__ dS, float* __restrict__ dgamma) {
    extern __shared__ float sm[];
    const int PQ3 = p.Pq * 3, PV3 = p.Pv * 3;
    const int N = p.N, H = p.H, C = p.C, Cp = p.Cp;
    const int CW = C + PV3;                            // staged key-side channels: v | value points
    float* s_q = sm;                                   // [32][PQ3]
    float* s_k = s_q + B1_TI * PQ3;                    // [32][PQ3+1]
    float* s_do = s_k + TJ * (PQ3 + 1);                // [CW + Cp][32]   channel-major dO rows of the tile
    float* s_v = s_do + (CW + Cp) * B1_TI;             // [32][CW+1]      key-side values of the tile
    __shared__ float s_red[8];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int i0 = blockIdx.x * B1_TI, h = blockIdx.y, f = blockIdx.z;
    const int D = concat_width(p);
    const int HPv = H * p.Pv;
    const int offPair = H * C + 4 * HPv;

    for (int e = tid; e < B1_TI * PQ3; e += 256) {
        const int r = e / PQ3, c = e % PQ3;
        const int i = i0 + r;
        s_q[e] = (i < N) ? p.q_pts[(((long)f * N + i) * H + h) * PQ3 + c] : 0.f;
    }
    for (int e = tid; e < (CW + Cp) * B1_TI; e += 256) {
        const int r = e % B1_TI, c = e / B1_TI;
        const int i = i0 + r;
        float v = 0.f;
        if (i < N) {
            const long fr = (long)f * N + i;
            if (c < C) v = dcat[fr * D + h * C + c];
            else if (c < CW) v = d_og[(fr * H + h) * PV3 + (c - C)];
            else v = dcat[fr * D + offPair + h * Cp + (c - CW)];
        }
        s_do[c * B1_TI + r] = v;
    }
    const float gam = -0.5f * p.gamma[h];
    const float* l0 = p.logit0 + (long)f * p.l_fs + (long)h * N * N;
    const float* vbase = p.kv + (long)f * p.kv_fs + (long)h * 2 * C + C;
    const float* kvp = p.kv_pts + (long)f * N * H * (PQ3 + PV3) + (long)h * (PQ3 + PV3);
    const float* zbase = p.pair + (long)f * p.pair_fs;
    const float* mrow = p.mask + (long)f * N;
    float lse_r[B1_RB], dl_r[B1_RB];
#pragma unroll
    for (int r = 0; r < B1_RB; ++r) {
        const int i = i0 + warp * B1_RB + r;
        lse_r[r] = (i < N) ? p.lse[((long)f * H + h) * N + i] : 0.f;
        dl_r[r] = (i < N) ? delta[((long)f * H + h) * N + i] : 0.f;
    }
    float dgam = 0.f;
    for (int j0 = 0; j0 < N; j0 += TJ) {
        __syncthreads();
        for (int e = tid; e < TJ * PQ3; e += 256) {
            const int jj = e / PQ3, c = e % PQ3;
            const int j = j0 + jj;
            s_k[jj * (PQ3 + 1) + c] = (j < N) ? kvp[(long)j * H * (PQ3 + PV3) + c] : 0.f;
        }
        for (int e = tid; e < TJ * CW; e += 256) {
            const int jj = e / CW, c = e % CW;
            const int j = j0 + jj;
            float v = 0.f;
            if (j < N) v = (c < C) ? vbase[(long)j * H * 2 * C + c] : kvp[(long)j * H * (PQ3 + PV3) + PQ3 + (c - C)];
            s_v[jj * (CW + 1) + c] = v;
        }
        __syncthreads();
        const int j = j0 + lane;
        float dP[B1_RB] = {0.f, 0.f, 0.f, 0.f};
        const float* vr = s_v + lane * (CW + 1);
        for (int c = 0; c < CW; ++c) {
            const float v = vr[c];
            const float4 g = *reinterpret_cast<const float4*>(s_do + c * B1_TI + warp * B1_RB);
            dP[0] = fmaf(g.x, v, dP[0]); dP[1] = fmaf(g.y, v, dP[1]); dP[2] = fmaf(g.z, v, dP[2]); dP[3] = fmaf(g.w, v, dP[3]);
        }
#pragma unroll
        for (int r = 0; r < B1_RB; ++r) {
            const int i = i0 + warp * B1_RB + r;
            float pv = 0.f, ds = 0.f;
            if (i < N && j < N) {
                const float* zr = zbase + ((long)i * N + j) * Cp;
                float dpz = 0.f;
                for (int c = 0; c < Cp; c += 4) {
                    const float4 z = __ldg(reinterpret_cast<const float4*>(zr + c));
                    dpz = fmaf(s_do[(CW + c) * B1_TI + warp * B1_RB + r], z.x, dpz);
                    dpz = fmaf(s_do[(CW + c + 1) * B1_TI + warp * B1_RB + r], z.y, dpz);
                    dpz = fmaf(s_do[(CW + c + 2) * B1_TI + warp * B1_RB + r], z.z, dpz);
                    dpz = fmaf(s_do[(CW + c + 3) * B1_TI + warp * B1_RB + r], z.w, dpz);
                }
                float d2 = 0.f;
                const float* qp = s_q + (warp * B1_RB + r) * PQ3;
                const float* kp = s_k + lane * (PQ3 + 1);
                for (int c = 0; c < PQ3; ++c) { const float d = qp[c] - kp[c]; d2 = fmaf(d, d, d2); }
                const float s = l0[(long)i * N + j] + gam * d2 + p.inf * (mrow[i] * mrow[j] - 1.f);
                pv = expf(s - lse_r[r]);
                ds = pv * (dP[r] + dpz - dl_r[r]);
                dgam = fmaf(ds, -0.5f * d2, dgam);
                const long o = (((long)h * p.F + f) * N + i) * N + j;
                Pm[o] = pv;
                dS[o] = ds;
            }
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

// B3: point gradients from the materialised dS.
//   dq_pts[f,i,h,c] = -gamma_h * sum_j dS[h,f,i,j] (qp[f,i,h,c] - kp[f,j,h,c])       (row pass,  transpose = 0)
//   dk_pts[f,j,h,c] = +gamma_h * sum_i dS[h,f,i,j] (qp[f,i,h,c] - kp[f,j,h,c])       (col pass,  transpose = 1)
// One warp per (f, h, row-or-column); lanes stride over the reduced index; PQ3 accumulators reduced by shuffles.
template <int MAXC>
__global__ void ipa_bwd_pts_kernel(const IpaParams p, const float* __restrict__ dS, float* __restrict__ dq_pts,
                                   float* __restrict__ dkv_pts, int transpose) {
    const int PQ3 = p.Pq * 3, PV3 = p.Pv * 3;
    const int N = p.N, H = p.H;
    const long wid = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (wid >= (long)p.F * H * N) return;
    const int lane = threadIdx.x & 31;
    const int a = (int)(wid % N);
    const int h = (int)((wid / N) % H);
    const int f = (int)(wid / ((long)N * H));
    const float gam = p.gamma[h];
    const float* qp = p.q_pts + ((long)f * N * H + h) * PQ3;                       // + i*H*PQ3
    const float* kp = p.kv_pts + ((long)f * N * H + h) * (PQ3 + PV3);              // + j*H*(PQ3+PV3)
    const float* ds = dS + ((long)h * p.F + f) * N * N;
    float self[MAXC], acc[MAXC];
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
        acc[c] = 0.f;
        self[c] = (c < PQ3) ? (transpose ? kp[(long)a * H * (PQ3 + PV3) + c] : qp[(long)a * H * PQ3 + c]) : 0.f;
    }
    for (int b = lane; b < N; b += 32) {
        const float w = transpose ? ds[(long)b * N + a] : ds[(long)a * N + b];
        const float* other = transpose ? qp + (long)b * H * PQ3 : kp + (long)b * H * (PQ3 + PV3);
#pragma unroll
        for (int c = 0; c < MAXC; ++c)
            if (c < PQ3) {
                const float diff = transpose ? (other[c] - self[c]) : (self[c] - other[c]);   // always qp - kp
                acc[c] = fmaf(w, diff, acc[c]);
            }
    }
#pragma unroll
    for (int c = 0; c < MAXC; ++c) acc[c] = warp_sum(acc[c]);
    if (lane == 0) {
        if (!transpose) {
            float* dst = dq_pts + (((long)f * N + a) * H + h) * PQ3;
            for (int c = 0; c < PQ3; ++c) dst[c] = -gam * acc[c];
        } else {
            float* dst = dkv_pts + (((long)f * N + a) * H + h) * (PQ3 + PV3);
            for (int c = 0; c < PQ3; ++c) dst[c] = gam * acc[c];
        }
    }
}

int fill_geometry(IpaParams& p) {
    DFOLD_REQUIRE(p.C % 4 == 0 && p.Cp % 4 == 0, "ipa: C (%d) and pair width (%d) must be multiples of 4", p.C, p.Cp);
    p.C4 = p.C / 4;
    p.P4 = (p.Pv * 3 + 3) / 4;
    p.Z4 = p.Cp / 4;
    const int tot = p.C4 + p.P4 + p.Z4;
    p.CGP = ((tot + 31) / 32) * 32;
    DFOLD_REQUIRE(p.CGP <= 512, "ipa: per-head channel count too large (%d groups)", tot);
    p.RG = 384 / p.CGP;
    if (p.RG < 1) p.RG = 1;
    if (p.RG > 8) p.RG = 8;
    return 0;
}

}  // namespace
}  // namespace dfold

using namespace dfold;

#define IPA_ARGS                                                                                                     \
    const float *logit0, long logit0_fstride, const float *kv, long kv_fstride, const float *q_pts,                  \
        const float *kv_pts, const float *pair, long pair_fstride, const float *quat, const float *trans,            \
        const float *mask, const float *gamma, int F, int N, int H, int C, int Pq, int Pv, int Cp, int dfold,        \
        float inf, float eps

static int make_params(IpaParams& p, IPA_ARGS) {
    p.logit0 = logit0; p.l_fs = logit0_fstride; p.kv = kv; p.kv_fs = kv_fstride; p.q_pts = q_pts; p.kv_pts = kv_pts;
    p.pair = pair; p.pair_fs = pair_fstride; p.quat = quat; p.trans = trans; p.mask = mask; p.gamma = gamma;
    p.out = nullptr; p.lse = nullptr;
    p.F = F; p.N = N; p.H = H; p.C = C; p.Pq = Pq; p.Pv = Pv; p.Cp = Cp; p.dfold = dfold; p.inf = inf; p.eps = eps;
    DFOLD_REQUIRE(F > 0 && N > 0 && H > 0 && Pq > 0 && Pv > 0, "ipa: empty problem");
    return fill_geometry(p);
}

extern "C" int dfold_ipa_attn_fwd(IPA_ARGS, float* out_cat, float* lse, void* stream) {
    IpaParams p;
    if (make_params(p, logit0, logit0_fstride, kv, kv_fstride, q_pts, kv_pts, pair, pair_fstride, quat, trans, mask, gamma,
                    F, N, H, C, Pq, Pv, Cp, dfold, inf, eps)) return 1;
    p.out = out_cat; p.lse = lse;
    const int TI = p.RG * RT;
    const int PQ3 = Pq * 3, PV3 = Pv * 3;
    const int SW = (TJ + 1 > PV3) ? TJ + 1 : PV3;
    const size_t smem = sizeof(float) * (size_t)(TI * PQ3 + TJ * (PQ3 + 1) + TI * SW + TJ * TI + 3 * TI);
    DFOLD_REQUIRE(smem <= 48 * 1024, "ipa_fwd: shared memory %zu exceeds 48 KB", smem);
    dim3 grid((unsigned)cdiv(N, TI), (unsigned)H, (unsigned)F);
    ipa_fwd_kernel<<<grid, p.CGP * p.RG, smem, as_stream(stream)>>>(p);
    return check_launch("ipa_fwd_kernel");
}

// workspaces: d_og [F,N,H,Pv,3], delta [F,H,N], P and dS [H,F,N,N]; outputs dq_pts [F,N,H,Pq,3], dkv_pts (k part only,
// [F,N,H,Pq+Pv,3] stride), dquat/dtrans from the epilogue, dgamma [H] (must be zeroed by the caller).
extern "C" int dfold_ipa_attn_bwd(IPA_ARGS, const float* out_cat, const float* lse, const float* dcat,
                                  float* d_og, float* delta, float* Pm, float* dS, float* dq_pts, float* dkv_pts,
                                  float* dquat, float* dtrans, float* dgamma, void* stream) {
    IpaParams p;
    if (make_params(p, logit0, logit0_fstride, kv, kv_fstride, q_pts, kv_pts, pair, pair_fstride, quat, trans, mask, gamma,
                    F, N, H, C, Pq, Pv, Cp, dfold, inf, eps)) return 1;
    p.lse = const_cast<float*>(lse);
    cudaStream_t st = as_stream(stream);
    ipa_bwd_pre_kernel<<<(unsigned)cdiv((long)F * N, 8), 256, 0, st>>>(p, out_cat, dcat, d_og, delta, dquat, dtrans);
    if (check_launch("ipa_bwd_pre_kernel")) return 1;
    const int PQ3 = Pq * 3, PV3 = Pv * 3, CW = C + PV3;
    const size_t smem = sizeof(float) * (size_t)(B1_TI * PQ3 + TJ * (PQ3 + 1) + (CW + Cp) * B1_TI + TJ * (CW + 1));
    static SmemCfg cfg;
    if (ensure_dyn_smem(ipa_bwd_row_kernel, smem, cfg, "ipa_bwd_row_kernel")) return 1;
    dim3 grid((unsigned)cdiv(N, B1_TI), (unsigned)H, (unsigned)F);
    ipa_bwd_row_kernel<<<grid, 256, smem, st>>>(p, dcat, d_og, delta, Pm, dS, dgamma);
    if (check_launch("ipa_bwd_row_kernel")) return 1;
    DFOLD_REQUIRE(PQ3 <= 48, "ipa_bwd: more than 16 query points per head are not supported");
    const unsigned blocks = (unsigned)cdiv((long)F * H * N, 8);
    if (PQ3 <= 12) {
        ipa_bwd_pts_kernel<12><<<blocks, 256, 0, st>>>(p, dS, dq_pts, dkv_pts, 0);
        ipa_bwd_pts_kernel<12><<<blocks, 256, 0, st>>>(p, dS, dq_pts, dkv_pts, 1);
    } else if (PQ3 <= 24) {
        ipa_bwd_pts_kernel<24><<<blocks, 256, 0, st>>>(p, dS, dq_pts, dkv_pts, 0);
        ipa_bwd_pts_kernel<24><<<blocks, 256, 0, st>>>(p, dS, dq_pts, dkv_pts, 1);
    } else {
        ipa_bwd_pts_kernel<48><<<blocks, 256, 0, st>>>(p, dS, dq_pts, dkv_pts, 0);
        ipa_bwd_pts_kernel<48><<<blocks, 256, 0, st>>>(p, dS, dq_pts, dkv_pts, 1);
    }
    return check_launch("ipa_bwd_pts_kernel");
}

// Epilogue-only backward (used by the tensor-core decomposition, csrc/ipa_v2.cu): d_og [F,N,H,Pv,3], delta [F,H,N],
// dquat [F,N,4], dtrans [F,N,3] from the concat buffer and its gradient.
extern "C" int dfold_ipa_pre_bwd(const float* quat, const float* trans, int F, int N, int H, int C, int Pv, int Cp, int dfold,
                                 const float* out_cat, const float* dcat, float* d_og, float* delta, float* dquat, float* dtrans,
                                 void* stream) {
    DFOLD_REQUIRE(F > 0 && N > 0 && H > 0, "dfold_ipa_pre_bwd: empty problem");
    IpaParams p{};
    p.quat = quat; p.trans = trans; p.F = F; p.N = N; p.H = H; p.C = C; p.Pv = Pv; p.Cp = Cp; p.dfold = dfold; p.Pq = 1;
    ipa_bwd_pre_kernel<<<(unsigned)cdiv((long)F * N, 8), 256, 0, as_stream(stream)>>>(p, out_cat, dcat, d_og, delta, dquat, dtrans);
    return check_launch("ipa_bwd_pre_kernel");
}
