// Fused invariant-point-attention forward core for the frame-shared (DFOLDv2) case, sm_90a.
//
// One CTA = (32 query residues, one trajectory frame, all 8 heads), 16 warps.  Per CTA, over key tiles of 32 residues:
//   pass 1   exact softmax statistics (row max m, row sum l) of
//                s[h,i,j] = logit0[h,i,j] - gamma_h/2 * sum_p |q_p(i) - k_p(j)|^2 + inf * (mask_i mask_j - 1)
//            with the coordinate differences in exact fp32: key points arrive by TMA (double-buffered tiles), each lane
//            keeps one key in registers, the query points are broadcast from shared memory, (m, l) are kept online per
//            lane and combined by warp shuffles at the end -- no whole-row shared memory, no cap on N;
//   pass 2   per key tile: (A) p = exp(s - m) / l, written once to shared memory (fp32, all heads) and to the bf16
//            hi/lo planes P[F,H,N,ldp]; (B1) pair aggregation o_pair[i,h,:] += p[h,i,j] z[i,j,:] with lanes across the
//            pair channels, z read once from L2 for all 8 heads; (B2) value-point aggregation
//            o_pt[h,i,:] += p[h,i,j] v_pts[j,h,:] with the tile's value points landing as one TMA box;
//   epilogue local-frame transform R_i^T (o_pt - t_i), norms, reference concat layout, coalesced stores.
// The scalar values O = P V are left to dfold_gemm_bf16x3_batched over the probability planes: one CTA's accumulator
// (8 heads x 256 channels x 32 rows in fp32 = 256 KB) fits neither the register file next to the 16 warps' state nor
// shared memory on sm_90.
//
// Reference: src/model/ipa_pytorch_dynamic.py:402-504 (logits :402-447, softmax :448, aggregations :455-504).
#include <cuda.h>
#include <stdlib.h>
#include "common.cuh"

namespace dfold {
namespace {

typedef unsigned long long u64;

constexpr int FH = 8;        // heads
constexpr int FTI = 32;      // query rows per CTA
constexpr int FTJ = 32;      // keys per tile
constexpr int FPQ = 8;       // query / key points
constexpr int FPV = 12;      // value points
constexpr int FCP = 32;      // pair channels (c_z / 4)
constexpr int PQ3 = FPQ * 3; // 24
constexpr int PV3 = FPV * 3; // 36
constexpr int FW = PQ3 + PV3;
constexpr int SPS = FH * FTJ + 4;      // row stride of the probability tile (floats): 16-byte aligned, odd in 16-byte units
constexpr int NCOMP = 512;             // 16 compute warps: (head, row half) in phase A, 2 rows in B1, (head, point half) in B2
constexpr int RH = FTI / 2;            // rows per warp in phase A
constexpr float LOG2E = 1.4426950408889634f;

struct FusedParams {
    const float* logit0;                   // [H,N,N]  frame-shared scalar logits (q.k / sqrt(3C) + b / sqrt(3))
    const float* q_pts;                    // [F,N,H,Pq,3]
    const float* kv_pts;                   // [F,N,H,Pq+Pv,3]
    const float* pair;                     // [N,N,Cp]
    const float* quat; const float* trans; // [F,N,4], [F,N,3]
    const float* mask;                     // [F,N]
    const float* gamma;                    // [H]
    uint16_t* p_hi; uint16_t* p_lo; long ldp;   // [F,H,N,ldp] or null
    float* cat;                            // [F,N,D]
    int F, N, C, dfold;
    float inf, eps;
    long long* stats;                      // development aid (dfold_debug_ipa_stats): 16 x int64 cycle counters per CTA
    int skip;                              // development knob (DFOLD_IPA_DEBUG_SKIP): bit 0 pass 1, 1 distances, 2 B1, 3 B2
};

__device__ __forceinline__ u64 pack2(float a, float b) { u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b)); return r; }
__device__ __forceinline__ void unpack2(u64 v, float& a, float& b) { asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); }
// coordinate pairs held as 64-bit words; sm_90 has no packed FP32 arithmetic, so each pair op is two scalar rn ops
__device__ __forceinline__ u64 sub2(u64 a, u64 b) {
    float a0, a1, b0, b1;
    unpack2(a, a0, a1); unpack2(b, b0, b1);
    return pack2(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
    float a0, a1, b0, b1, c0, c1;
    unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(c, c0, c1);
    return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ float ex2f(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ void comp_sync() { asm volatile("bar.sync 1, 512;" ::: "memory"); }   // the 16 warps

// ---- TMA / mbarrier wrappers (same forms as csrc/gemm_sm90.cu) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(bar) : "memory");
}
// squared distance summed over the 8 point pairs: q (shared memory, broadcast) against the lane's key in registers
__device__ __forceinline__ float dist2(const ulonglong2* __restrict__ q2, const u64 (&k)[12]) {
    ulonglong2 qq[6];
#pragma unroll
    for (int c = 0; c < 6; ++c) qq[c] = q2[c];                 // all six LDS.128 in flight before the first use
    u64 a0 = 0ull;
#pragma unroll
    for (int c = 0; c < 6; ++c) {
        const u64 d0 = sub2(qq[c].x, k[2 * c]);
        const u64 d1 = sub2(qq[c].y, k[2 * c + 1]);
        a0 = fma2(d0, d0, a0);
        a0 = fma2(d1, d1, a0);
    }
    float x0, x1;
    unpack2(a0, x0, x1);
    return x0 + x1;
}

__device__ __forceinline__ void load_key_global(const float* __restrict__ kv_pts, long fN, int jc, int h, u64 (&k)[12]) {
    const ulonglong2* src = reinterpret_cast<const ulonglong2*>(kv_pts + ((fN + jc) * FH + h) * FW);
#pragma unroll
    for (int c = 0; c < 6; ++c) {
        const ulonglong2 v = __ldg(src + c);
        k[2 * c] = v.x;
        k[2 * c + 1] = v.y;
    }
}
// this lane's key of the staged tile  s_k[h][j][24]
__device__ __forceinline__ void load_key(const float* __restrict__ s_k, int h, int lane, u64 (&k)[12]) {
    const ulonglong2* src = reinterpret_cast<const ulonglong2*>(s_k + (h * FTJ + lane) * PQ3);
#pragma unroll
    for (int c = 0; c < 6; ++c) {
        const ulonglong2 v = src[c];
        k[2 * c] = v.x;
        k[2 * c + 1] = v.y;
    }
}

// ---- shared memory plan (floats unless noted) ----
constexpr int kSQ = FH * FTI * PQ3;            // query points          [h][i][24]
constexpr int kSV = FTJ * FH * PV3;            // value points of a tile [j][h][36], written by ONE TMA box per tile
constexpr int kSP = FTI * SPS;                 // probabilities         [i][hp][j][2]
constexpr int kSRow = 2 * FTI;                 // per row {clamped row * N (int), mask_i * inf}
constexpr int kSStat = 2 * FH * FTI;           // per (h, row) {m, 1 / l}
constexpr int SST = 772;                       // staging row stride (floats): 16-byte aligned, 4-way instead of 32-way conflicts
constexpr int kStage = FTI * SST;              // epilogue staging of the point features
constexpr int kSK = FTJ * FH * PQ3;             // key points of a tile [h][j][24] (8 TMA boxes): pass 1, in the s_v / s_p space
constexpr int kWork = kSQ + kSV + kSP;
// [max(work, stage) | row | stat | barriers]: the epilogue stages in the work space
constexpr int kWorkFloats = kWork > kStage + FH * FTI * PV3 ? kWork : kStage + FH * FTI * PV3;
constexpr int kFusedBytes = 4 * (kWorkFloats + kSRow + kSStat) + 64 + 1024;      // + barriers + alignment slack

__global__ void __launch_bounds__(NCOMP, 1)
ipa_fused_fwd_kernel(const FusedParams p, const __grid_constant__ CUtensorMap map_pts, const __grid_constant__ CUtensorMap map_kpt) {
    extern __shared__ __align__(16) unsigned char sm_raw[];
    unsigned char* sm_base = sm_raw;
    sm_base = sm_raw + ((1024u - (smem_u32(sm_raw) & 1023u)) & 1023u);      // TMA boxes want 128 B alignment
    float* smf = reinterpret_cast<float*>(sm_base);
    float* s_q = smf;
    float* s_v = s_q + kSQ;
    float* s_p = s_v + kSV;
    float* s_row = smf + kWorkFloats;
    float* s_stat = s_row + kSRow;
    float* stage = smf;
    const uint32_t bar_u32 = smem_u32(s_stat + kSStat);
    const uint32_t vfull_bar = bar_u32;                                      // value-point tile landed
    auto kfull_bar = [&](int b) { return bar_u32 + 8u * (1 + b); };         // key-point tiles of pass 1 (two buffers)

    const int N = p.N;
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);      // provably warp-uniform
    const int i0 = blockIdx.x * FTI, f = blockIdx.y;
    const long fN = (long)f * N;
    const int ntiles = (N + FTJ - 1) / FTJ;

    {
        // =============================== compute warps ===============================
        const int h = warp & 7;                                  // phase A / B2: this warp's head
        const int wh = warp >> 3;                                // phase A: row half, B2: key half
        const int rbase = wh * RH;
        // ---- query points of the 32 rows, all heads: s_q[h][i][24];  per-row constants ----
        for (int e = tid; e < FTI * FH * (PQ3 / 4); e += NCOMP) {
            const int c4 = e % (PQ3 / 4), hh = (e / (PQ3 / 4)) % FH, r = e / (FH * (PQ3 / 4));
            const int i = i0 + r;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < N) v = __ldg(reinterpret_cast<const float4*>(p.q_pts + ((fN + i) * FH + hh) * PQ3) + c4);
            reinterpret_cast<float4*>(s_q + (hh * FTI + r) * PQ3)[c4] = v;
        }
        if (tid == 32) {
            mbar_init(vfull_bar, 1);
            for (int b = 0; b < 2; ++b) mbar_init(kfull_bar(b), 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        if (tid < FTI) {
            const int ic = min(i0 + tid, N - 1);
            reinterpret_cast<int*>(s_row)[2 * tid] = ic * N;
            s_row[2 * tid + 1] = __ldg(p.mask + fN + ic) * p.inf;
        }
        const float gam = -0.5f * __ldg(p.gamma + h);
        const float ninf = -p.inf;
        const float* l0h = p.logit0 + (long)h * N * N;
        const float* mrow = p.mask + fN;
        const ulonglong2* q2 = reinterpret_cast<const ulonglong2*>(s_q + (h * FTI + rbase) * PQ3);
        const float2* rowc = reinterpret_cast<const float2*>(s_row) + rbase;
        comp_sync();
        const bool timing = p.stats != nullptr && tid == 0;
        long long tc0 = timing ? clock64() : 0, c_p1 = 0, c_a = 0, c_b1 = 0, c_b2 = 0, c_sync = 0, c_epi = 0;

        // =============================== pass 1: softmax statistics ===============================
        // key tiles arrive by TMA (8 boxes of 24 coordinates x 32 residues, one per head), double-buffered in the s_v / s_p
        // space that pass 2 uses later: the key points are read from L2 once per CTA and pass
        auto issue_keys = [&](float* dst, uint32_t bar, int j0) {
            mbar_expect_tx(bar, kSK * 4);
#pragma unroll
            for (int hh = 0; hh < FH; ++hh) tma_load_3d(smem_u32(dst + hh * FTJ * PQ3), &map_kpt, bar, 0, hh, (int)(fN + j0));
        };
        {
            const int nt1 = (p.skip & 1) ? 0 : ntiles;
            if (tid == 0) {
                if (nt1 > 0) issue_keys(s_v, kfull_bar(0), 0);
                if (nt1 > 1) issue_keys(s_p, kfull_bar(1), FTJ);
            }
            float m[RH], l[RH];
#pragma unroll
            for (int rr = 0; rr < RH; ++rr) { m[rr] = -3.0e38f; l[rr] = 0.f; }
#pragma unroll 1
            for (int t = 0; t < nt1; ++t) {
                const int j = t * FTJ + lane;
                const bool jok = j < N;
                const int jc = min(j, N - 1);
                const float mj = jok ? __ldg(mrow + jc) : 0.f;
                float l0r[RH];
#pragma unroll
                for (int rr = 0; rr < RH; ++rr) l0r[rr] = __ldg(l0h + __float_as_int(rowc[rr].x) + jc);
                mbar_wait(kfull_bar(t & 1), (t >> 1) & 1);
                u64 k[12];
                load_key((t & 1) ? s_p : s_v, h, lane, k);
#pragma unroll
                for (int rr = 0; rr < RH; ++rr) {
                    const float d2 = dist2(q2 + rr * (PQ3 / 4), k);
                    float s = fmaf(gam, d2, l0r[rr]) + fmaf(rowc[rr].y, mj, ninf);
                    s = jok ? s : -1.0e30f;
                    // online (m, l) with one exponential: e = exp(-|s - m|)
                    const float e = ex2f(-fabsf(s - m[rr]) * LOG2E);
                    const bool up = s > m[rr];
                    l[rr] = up ? fmaf(l[rr], e, 1.f) : l[rr] + e;
                    m[rr] = up ? s : m[rr];
                }
                comp_sync();                                          // every warp has its keys of this buffer in registers
                if (tid == 0 && t + 2 < nt1) issue_keys((t & 1) ? s_p : s_v, kfull_bar(t & 1), (t + 2) * FTJ);
            }
#pragma unroll
            for (int rr = 0; rr < RH; ++rr) {
                const float M = warp_max(m[rr]);
                const float L = warp_sum(l[rr] * ex2f((m[rr] - M) * LOG2E));
                if (lane == rr) {
                    s_stat[2 * (h * FTI + rbase + rr)] = M;
                    s_stat[2 * (h * FTI + rbase + rr) + 1] = 1.f / L;
                }
            }
        }
        comp_sync();
        if (timing) { c_p1 = clock64() - tc0; }

        // =============================== pass 2: probabilities and aggregations ===============================
        u64 accp[2][4];                      // pair aggregation: [row of this warp][head pair] x this lane's channel
#pragma unroll
        for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) accp[a][b] = 0ull;
        u64 accv[10];                        // value points: (head, coordinate half = warp, row = lane) x 20 | 16 coordinates
#pragma unroll
        for (int c = 0; c < 10; ++c) accv[c] = 0ull;

        const int hp = h >> 1, hodd = h & 1;
        const float2* statc = reinterpret_cast<const float2*>(s_stat) + h * FTI + rbase;
        float* sp_w = s_p + rbase * SPS + hp * (2 * FTJ) + lane * 2 + hodd;
        const int nrow_ok = max(0, min(RH, N - i0 - rbase));           // valid rows of this warp's half
        uint16_t* ph = p.p_hi + ((long)(f * FH + h) * N + i0 + rbase) * p.ldp;
        uint16_t* pl = p.p_lo + ((long)(f * FH + h) * N + i0 + rbase) * p.ldp;

        for (int t = 0; t < ntiles; ++t) {
            const int j0 = t * FTJ;
            // value points of this tile -> s_v[j][h][36]: one TMA box (36 coordinates x 8 heads x 32 residues) of the fp32
            // [F*N][H][60] point tensor; rows past the end of the tensor are zero-filled, rows of the next frame meet p = 0
            if (tid == 0) {
                mbar_expect_tx(vfull_bar, kSV * 4);
                tma_load_3d(smem_u32(s_v), &map_pts, vfull_bar, PQ3, 0, (int)(fN + j0));
            }
            // ---- phase A: warp = (head, row half), lane = key ----
            long long tt = timing ? clock64() : 0;
            {
                const int j = j0 + lane;
                const bool jok = j < N;
                const int jc = min(j, N - 1);
                const float mj = jok ? __ldg(mrow + jc) : 0.f;
                u64 k[12];
                load_key_global(p.kv_pts, fN, jc, h, k);
#pragma unroll 1
                for (int rb = 0; rb < RH; rb += 8) {
                    const float2* rowb = rowc + rb;
                    const float2* statb = statc + rb;
                    const ulonglong2* qb = q2 + rb * (PQ3 / 4);
                    float* spb = sp_w + rb * SPS;
                    uint16_t* phb = ph + (long)rb * p.ldp + j;
                    uint16_t* plb = pl + (long)rb * p.ldp + j;
                    const int nok = nrow_ok - rb;
                    float l0r[8];
#pragma unroll
                    for (int rr = 0; rr < 8; ++rr) l0r[rr] = __ldg(l0h + __float_as_int(rowb[rr].x) + jc);
#pragma unroll
                    for (int rr = 0; rr < 8; ++rr) {
                        const float2 rc = rowb[rr];
                        const float2 st = statb[rr];
                        const float d2 = (p.skip & 2) ? 1.f : dist2(qb + rr * (PQ3 / 4), k);
                        const float s = fmaf(gam, d2, l0r[rr]) + fmaf(rc.y, mj, ninf);
                        float pv = ex2f((s - st.x) * LOG2E) * st.y;      // (s - m) first: exact for the terms that matter
                        pv = jok ? pv : 0.f;
                        spb[rr * SPS] = pv;
                        const __nv_bfloat16 bh = __float2bfloat16_rn(pv);
                        const __nv_bfloat16 bl = __float2bfloat16_rn(pv - __bfloat162float(bh));
                        if (jok && rr < nok) {
                            *phb = __bfloat16_as_ushort(bh);
                            *plb = __bfloat16_as_ushort(bl);
                        }
                        phb += p.ldp; plb += p.ldp;
                    }
                }
            }
            if (timing) { const long long n = clock64(); c_a += n - tt; tt = n; }
            comp_sync();
            if (timing) { const long long n = clock64(); c_sync += n - tt; tt = n; }
            // ---- phase B1: pair aggregation, warp = 2 rows, lane = pair channel ----
            if (!(p.skip & 4)) {
                // eight batches of 8 keys (2 rows x 4 quarters of the tile); the z loads of batch b + 1 are in flight while
                // batch b is accumulated (L2 latency, not bandwidth, bounds this phase)
                const bool full = j0 + FTJ <= N;
                const float* zrow0 = p.pair + ((long)__float_as_int(s_row[4 * warp]) + j0) * FCP + lane;
                const float* zrow1 = p.pair + ((long)__float_as_int(s_row[4 * warp + 2]) + j0) * FCP + lane;
                auto load_z = [&](int bt, float (&z)[8]) {
                    const float* zr = (bt >> 2) ? zrow1 : zrow0;
                    const int jb = (bt & 3) * 8;
                    if (full) {
#pragma unroll
                        for (int q = 0; q < 8; ++q) z[q] = __ldg(zr + (jb + q) * FCP);
                    } else {
#pragma unroll
                        for (int q = 0; q < 8; ++q) z[q] = __ldg(zr + (min(j0 + jb + q, N - 1) - j0) * FCP);
                    }
                };
                float zc[8], zn[8];
                load_z(0, zc);
#pragma unroll
                for (int bt = 0; bt < 8; ++bt) {
                    if (bt < 7) load_z(bt + 1, zn);
                    const int a = bt >> 2, jb = (bt & 3) * 8;
                    const float* prow = s_p + (warp * 2 + a) * SPS;
#pragma unroll
                    for (int q = 0; q < 8; q += 2) {
                        const u64 zz0 = pack2(zc[q], zc[q]), zz1 = pack2(zc[q + 1], zc[q + 1]);
                        ulonglong2 pp[4];
#pragma unroll
                        for (int b = 0; b < 4; ++b) pp[b] = *reinterpret_cast<const ulonglong2*>(prow + b * (2 * FTJ) + (jb + q) * 2);
#pragma unroll
                        for (int b = 0; b < 4; ++b) {
                            accp[a][b] = fma2(pp[b].x, zz0, accp[a][b]);
                            accp[a][b] = fma2(pp[b].y, zz1, accp[a][b]);
                        }
                    }
#pragma unroll
                    for (int q = 0; q < 8; ++q) zc[q] = zn[q];
                }
            }
            if (timing) { const long long n = clock64(); c_b1 += n - tt; tt = n; }
            // ---- phase B2: value points, warp = (head, coordinates 0..19 | 20..35), lane = row ----
            mbar_wait(vfull_bar, t & 1);
            if (!(p.skip & 8)) {
                const float* prow = s_p + lane * SPS + hp * (2 * FTJ);
                const float* vbase = s_v + h * PV3 + wh * 20;
#pragma unroll 4
                for (int jj = 0; jj < FTJ; jj += 2) {
                    const float4 pq = *reinterpret_cast<const float4*>(prow + jj * 2);    // (h0,h1)@jj, (h0,h1)@jj+1
                    const float pa = hodd ? pq.y : pq.x, pb = hodd ? pq.w : pq.z;
                    const u64 ppa = pack2(pa, pa), ppb = pack2(pb, pb);
                    const ulonglong2* va = reinterpret_cast<const ulonglong2*>(vbase + jj * (FH * PV3));
                    const ulonglong2* vb = reinterpret_cast<const ulonglong2*>(vbase + (jj + 1) * (FH * PV3));
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const ulonglong2 x = va[c];
                        accv[2 * c] = fma2(ppa, x.x, accv[2 * c]);
                        accv[2 * c + 1] = fma2(ppa, x.y, accv[2 * c + 1]);
                    }
                    if (wh == 0) {
                        const ulonglong2 x = va[4];
                        accv[8] = fma2(ppa, x.x, accv[8]);
                        accv[9] = fma2(ppa, x.y, accv[9]);
                    }
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const ulonglong2 x = vb[c];
                        accv[2 * c] = fma2(ppb, x.x, accv[2 * c]);
                        accv[2 * c + 1] = fma2(ppb, x.y, accv[2 * c + 1]);
                    }
                    if (wh == 0) {
                        const ulonglong2 x = vb[4];
                        accv[8] = fma2(ppb, x.x, accv[8]);
                        accv[9] = fma2(ppb, x.y, accv[9]);
                    }
                }
            }
            if (timing) { const long long n = clock64(); c_b2 += n - tt; tt = n; }
            comp_sync();
            if (timing) { const long long n = clock64(); c_sync += n - tt; tt = n; }
        }
        const long long te0 = timing ? clock64() : 0;

        // =============================== epilogue ===============================
        const int D = FH * (p.C + (p.dfold ? 8 : 4) * FPV + FCP);
        const int HPv = FH * FPV;
        const int offLoc = FH * p.C, offPair = offLoc + 4 * HPv, offG = offPair + FH * FCP;
        // pair features straight to the concat buffer (128-byte coalesced per (row, head))
#pragma unroll
        for (int a = 0; a < 2; ++a) {
            const int i = i0 + warp * 2 + a;
            if (i < N) {
                float* orow = p.cat + (fN + i) * D + offPair + lane;
#pragma unroll
                for (int b = 0; b < 4; ++b) {
                    float x, y;
                    unpack2(accp[a][b], x, y);
                    orow[(2 * b) * FCP] = x;
                    orow[(2 * b + 1) * FCP] = y;
                }
            }
        }
        // point features.  The coordinate halves meet in shared memory, s_x[h][row][36]; then thread (h, half, row) transforms
        // points 6 half .. 6 half + 5:  stage[i][0..384) = local xyz + norms, [384..768) = global xyz + norms
        comp_sync();                                                  // the work buffers are free
        float* s_x = stage + kStage;                                  // 9216 floats behind the staging rows
        {
            u64* dst = reinterpret_cast<u64*>(s_x + (h * FTI + lane) * PV3 + wh * 20);
#pragma unroll
            for (int c = 0; c < 8; ++c) dst[c] = accv[c];
            if (wh == 0) { dst[8] = accv[8]; dst[9] = accv[9]; }
        }
        comp_sync();
        {
            const int r = lane;
            const int ic = min(i0 + r, N - 1);
            const float4 q = __ldg(reinterpret_cast<const float4*>(p.quat + 4 * (fN + ic)));
            float R[9];
            quat_to_rot9(q.x, q.y, q.z, q.w, R);
            const float tx = __ldg(p.trans + 3 * (fN + ic)), ty = __ldg(p.trans + 3 * (fN + ic) + 1), tz = __ldg(p.trans + 3 * (fN + ic) + 2);
            float g[PV3 / 2];
            {
                const u64* src = reinterpret_cast<const u64*>(s_x + (h * FTI + lane) * PV3 + wh * 18);
#pragma unroll
                for (int c = 0; c < PV3 / 4; ++c) unpack2(src[c], g[2 * c], g[2 * c + 1]);
            }
            float* srow = stage + r * SST;
#pragma unroll
            for (int pt = 0; pt < FPV / 2; ++pt) {
                const float gx = g[3 * pt], gy = g[3 * pt + 1], gz = g[3 * pt + 2];
                const float x = gx - tx, y = gy - ty, z = gz - tz;
                const float lx = R[0] * x + R[3] * y + R[6] * z;
                const float ly = R[1] * x + R[4] * y + R[7] * z;
                const float lz = R[2] * x + R[5] * y + R[8] * z;
                const int kk = h * FPV + wh * (FPV / 2) + pt;
                srow[kk] = lx; srow[HPv + kk] = ly; srow[2 * HPv + kk] = lz;
                srow[3 * HPv + kk] = sqrtf(lx * lx + ly * ly + lz * lz + p.eps);
                srow[384 + kk] = gx; srow[384 + HPv + kk] = gy; srow[384 + 2 * HPv + kk] = gz;
                srow[384 + 3 * HPv + kk] = sqrtf(gx * gx + gy * gy + gz * gz + p.eps);
            }
        }
        comp_sync();
        {
            const int nseg = p.dfold ? 2 : 1;
            for (int e = tid; e < FTI * nseg * 96; e += NCOMP) {
                const int c4 = e % 96, sg = (e / 96) % nseg, r = e / (96 * nseg);
                const int i = i0 + r;
                if (i >= N) continue;
                const float4 v = *reinterpret_cast<const float4*>(stage + r * SST + sg * 384 + c4 * 4);
                float* dst = p.cat + (fN + i) * D + (sg ? offG : offLoc) + c4 * 4;
                *reinterpret_cast<float4*>(dst) = v;
            }
        }
        if (timing) {
            long long* st = p.stats + 16 * ((long)blockIdx.y * gridDim.x + blockIdx.x);
            c_epi = clock64() - te0;
            st[4] = clock64() - tc0; st[5] = c_p1; st[6] = c_a; st[7] = c_b1; st[8] = c_b2; st[9] = c_sync; st[10] = c_epi;
        }
    }
}

SmemCfg g_fused_cfg;
long long* g_ipa_stats = nullptr;      // set by dfold_debug_ipa_stats

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn fused_get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}
// fp32 point tensor [rows][H][60] viewed as (60, H, rows); box = 36 value coordinates x 8 heads x 32 residues, no swizzle
int fused_make_pts_map(CUtensorMap* m, const void* base, long rows) {
    EncodeTiledFn enc = fused_get_encode();
    DFOLD_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled unavailable (driver too old?)");
    DFOLD_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "ipa_fused_fwd: kv_pts must be 16-byte aligned");
    cuuint64_t dims[3] = {(cuuint64_t)FW, (cuuint64_t)FH, (cuuint64_t)rows};
    cuuint64_t strides[2] = {(cuuint64_t)FW * 4, (cuuint64_t)FH * FW * 4};
    cuuint32_t box[3] = {(cuuint32_t)PV3, (cuuint32_t)FH, (cuuint32_t)FTJ};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    DFOLD_REQUIRE(r == CUDA_SUCCESS, "ipa_fused_fwd: cuTensorMapEncodeTiled (points) failed (%d)", (int)r);
    return 0;
}

// the same tensor with the box of one head's key points: 24 coordinates x 1 head x 32 residues
int fused_make_key_map(CUtensorMap* m, const void* base, long rows) {
    EncodeTiledFn enc = fused_get_encode();
    DFOLD_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled unavailable (driver too old?)");
    cuuint64_t dims[3] = {(cuuint64_t)FW, (cuuint64_t)FH, (cuuint64_t)rows};
    cuuint64_t strides[2] = {(cuuint64_t)FW * 4, (cuuint64_t)FH * FW * 4};
    cuuint32_t box[3] = {(cuuint32_t)PQ3, 1, (cuuint32_t)FTJ};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    DFOLD_REQUIRE(r == CUDA_SUCCESS, "ipa_fused_fwd: cuTensorMapEncodeTiled (key points) failed (%d)", (int)r);
    return 0;
}

}  // namespace
}  // namespace dfold

using namespace dfold;

// Development aid: when `buf` (device, 16 x int64 per CTA of the next fused-IPA launches) is non-null the kernel records, per
// CTA, cycle counters of thread 0 ({total, pass 1, phase A, B1, B2, barriers, epilogue}) at slots 4-10.
extern "C" int dfold_debug_ipa_stats(long long* buf) {
    g_ipa_stats = buf;
    return 0;
}

// Fused forward core.  Writes the point and pair columns of the concat buffer and the bf16 hi/lo probability planes; the
// scalar-value columns [0, H*C) are left to dfold_gemm_bf16x3_batched over those planes.
// Shapes: H = 8, Pq = 8, Pv = 12, Cp = 32 (DFOLDv2 preset A); other shapes use dfold_ipa_attn_fwd.
extern "C" int dfold_ipa_fused_fwd(const float* logit0, const float* q_pts, const float* kv_pts, const float* pair,
                                   const float* quat, const float* trans, const float* mask, const float* gamma,
                                   uint16_t* p_hi, uint16_t* p_lo, long ldp,
                                   int F, int N, int H, int C, int Pq, int Pv, int Cp,
                                   int dfold, float inf, float eps, float* out_cat, void* stream) {
    DFOLD_REQUIRE(F > 0 && N > 0, "ipa_fused_fwd: empty problem");
    DFOLD_REQUIRE(H == FH && Pq == FPQ && Pv == FPV && Cp == FCP, "ipa_fused_fwd: built for H=8, Pq=8, Pv=12, Cp=32 (got %d, %d, %d, %d)", H, Pq, Pv, Cp);
    DFOLD_REQUIRE(p_hi != nullptr && p_lo != nullptr && ldp >= N, "ipa_fused_fwd: bad probability planes");
    DFOLD_REQUIRE(F <= 65535 && (long)N * N < (1l << 31), "ipa_fused_fwd: problem too large for one launch");
    FusedParams p;
    p.logit0 = logit0; p.q_pts = q_pts; p.kv_pts = kv_pts; p.pair = pair; p.quat = quat; p.trans = trans; p.mask = mask;
    p.gamma = gamma; p.p_hi = p_hi; p.p_lo = p_lo; p.ldp = ldp; p.cat = out_cat; p.F = F; p.N = N; p.C = C; p.dfold = dfold;
    p.inf = inf; p.eps = eps;
    { const char* e = getenv("DFOLD_IPA_DEBUG_SKIP"); p.skip = e ? atoi(e) : 0; }
    p.stats = g_ipa_stats;
    dim3 grid((unsigned)cdiv(N, FTI), (unsigned)F);
    CUtensorMap maps[2];
    memset(maps, 0, sizeof(maps));
    if (fused_make_pts_map(&maps[0], kv_pts, (long)F * N)) return 1;
    if (fused_make_key_map(&maps[1], kv_pts, (long)F * N)) return 1;
    if (ensure_dyn_smem(ipa_fused_fwd_kernel, kFusedBytes, g_fused_cfg, "ipa_fused_fwd")) return 1;
    ipa_fused_fwd_kernel<<<grid, NCOMP, kFusedBytes, as_stream(stream)>>>(p, maps[0], maps[1]);
    return check_launch("ipa_fused_fwd_kernel");
}
