// Split-precision (bf16 x 3) tensor-core GEMM / implicit 5x5 convolution for sm_90a.
//
//   C[m, n] = act(alpha * sum_{tap, k} A[m + off(tap), k] * B[tap][n][k] + bias[n]) + beta * R[m, n]
//
// fp32 operands are pre-split by `dfold_split2d` / `dfold_conv_weight_prep` into bf16 planes
// x = hi + lo (hi = bf16(x), lo = bf16(x - hi)); the kernel accumulates hi*hi + hi*lo + lo*hi in fp32, which keeps
// ~16 mantissa bits per operand (relative error ~2^-17 per product, vs 2^-11 for plain TF32/BF16 — SURVEY.md §0
// "precision trap").
//
// Structure (one CTA = one 128 x BN output tile, BN in {64, 128}, 384 threads = 3 warpgroups):
//   warpgroup 0    TMA producer (one thread): cp.async.bulk.tensor.3d (128B swizzle) of the A / B hi+lo tiles into a
//                  multi-stage smem ring; the 3-D tensor map of the activations makes the 5x5 halo an out-of-bounds
//                  zero fill, so the convolution needs no im2col and no padding buffer.
//   warpgroups 1-2 wgmma consumers, one 64-row half of the tile each: 3 products x 4 K-steps of m64nBNk16 per stage
//                  into a register accumulator.  The tensor core's fp32 accumulation is not round-to-nearest, and its
//                  error grows with the number of MMAs folded into one accumulator, so that accumulator only ever holds
//                  kChunk = 4 k-blocks (48 MMAs); it is then added into a second fp32 register accumulator with
//                  round-to-nearest CUDA-core adds.  Bias / activation / residual are applied on the way out.
//
// Replaces (reference file:line): nn.Linear in src/model/ipa_pytorch_dynamic.py:284-305,757-796,590,
// openfold/model/structure_module.py:102-110,58-59; nn.Conv2d stack src/model/ipa_pytorch_dynamic.py:664-706.
#include <cuda.h>
#include <stdlib.h>
#include "common.cuh"

namespace dfold {
namespace {

constexpr int BM = 128;
constexpr int BK = 64;          // 64 bf16 = 128 B = one swizzle row
constexpr int WG_K = 16;        // K of one wgmma
constexpr int NTHREADS = 384;   // producer warpgroup + 2 consumer warpgroups
constexpr int kChunk = 4;       // k-blocks accumulated by the tensor core before promotion to the fp32 accumulator

template <int BN> struct TileCfg {
    static_assert(BN == 64 || BN == 128, "tile width");
    static constexpr int kStages = (BN >= 128) ? 3 : 4;
    static constexpr int kABytes = BM * BK * 2;               // one plane
    static constexpr int kBBytes = BN * BK * 2;
    static constexpr int kStageBytes = 2 * kABytes + 2 * kBBytes;
    static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};

struct GemmParams {
    int mode;            // 0: A rows = (frame, residue) tiles, taps outer / K inner   1: wgrad (K = pixels)
    int num_kb;          // k-blocks per tile
    int kc;              // mode 0: k-chunks per tap; mode 1: residue blocks per frame
    int taps_n, taps_f;  // tap grid (1x1 for a plain linear)
    int tiles_per_frame; // mode 0: ceil(Nr / 128)
    int Nr;              // mode 0: residues per frame (rows per frame)
    long out_rows;       // valid rows of the output (mode 0: F*Nr, mode 1: M)
    int n_out;           // valid columns
    float* out; long ldo; long out_tap_stride;
    const float* bias;
    const float* res; long ldr;
    float alpha, beta;
    int act;             // 0 none, 1 relu, 2 silu
    // ---- batching (defaults describe the plain conv / linear case) ----
    // mode 0: the "frame" index f0 of a row tile doubles as a batch id: hb = f0 % bmod
    int bmod;            // >= 1
    int a_f_div;         // A frame coordinate            = f0 / a_f_div
    int a_k_bstride;     // A K-coordinate offset         = hb * a_k_bstride
    int b_k_ofs;         // B K-coordinate offset         = b_k_ofs + hb * b_k_bstride
    int b_k_bstride;
    int b_z_bstride;     // B third coordinate            = tap + hb * b_z_bstride
    int f_start;         // A frame coordinate offset (output frame f reads input frames f + f_start + df): cropped convs
    int b_f_add;         // mode 1: B outer coordinate offset
    int o_f_div;         // output row                    = (f0 / o_f_div) * Nr + n
    long o_col_bstride;  // output column offset          = hb * o_col_bstride
    // mode 1: blockIdx.z = zq (tap or batch id)
    int a_f_mul, a_z_mul;   // A outer coordinate = f * a_f_mul + zq * a_z_mul
    int b_f_mul, b_z_mul;   // B outer coordinate = f * b_f_mul + zq * b_z_mul (+ df)
    int b_n_zmul;           // B column offset    = zq * b_n_zmul
    // ---- stacked windows (0: 3-D operand maps, the plain path) ----
    // windows > 0: the activation maps gain a 4th (window) dimension; the frame halo is zero-filled at every window's edge.
    // mode 0: row tiles run window-major, win_tiles per window, output rows (w * F_out + f) * Nr + n.
    // mode 1: the k-blocks run window-major, win_kb per window.
    int windows;
    int win_tiles, win_fout, win_kb;
    long long* stats;       // debug (dfold_debug_gemm_stats): per CTA {total, consumer wait full, producer wait empty, 0} cycles
};

// ---------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
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
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
        ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar) : "memory");
}
// A / B tile load of the producer: 3-D maps, or with stacked windows 4-D maps whose outer coordinate is the window
__device__ __forceinline__ void tma_load(bool win, uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2,
                                         int w) {
    if (win) tma_load_4d(dst, map, bar, c0, c1, c2, w);
    else tma_load_3d(dst, map, bar, c0, c1, c2);
}

// 128B-swizzled operand tile descriptors (sm_90 wgmma layout: start >> 4 in [0,14), LBO in [16,30), SBO in [32,46),
// layout type in [62,64) with 1 = 128B swizzle).  Every tile base is 1024-byte aligned, so the base offset is 0.
// K-major: rows of 128 B (64 k), 8-row groups 1024 B apart (SBO); the LBO is unused.
__device__ __forceinline__ uint64_t make_sw128_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// MN-major (weight-gradient mode): the tile is stored [k][mn] with 64 mn-elements (128 B) contiguous per k row; 8 k-rows
// form a 1024 B swizzle atom (SBO), 64-wide mn atoms are 64 rows x 128 B = 8192 B apart (LBO).
__device__ __forceinline__ uint64_t make_sw128_mn_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)(8192 >> 4) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across a wgmma fence / wait
template <int R> __device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] B[16 x N], bf16 operands from shared memory, fp32 accumulator in registers.
// MN = 0: both operands K-major;  MN = 1: both MN-major (transposed).  scale_d = 0 overwrites D.
template <int N, int MN> __device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_bf16<64, 0>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, 0, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<64, 1>(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, %32, %33, p, 1, 1, 1, 1;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<128, 0>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, 0, 0;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_bf16<128, 1>(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, %64, %65, p, 1, 1, 1, 1;\n\t"
        "}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(scale_d));
}

template <int BN, int MN>
__device__ __forceinline__ void mma_stage(float (&part)[BN / 2], uint32_t sa_hi, uint32_t sa_lo, uint32_t sb_hi, uint32_t sb_lo,
                                          bool chunk_start) {
    const uint64_t da_hi = MN ? make_sw128_mn_desc(sa_hi) : make_sw128_desc(sa_hi);
    const uint64_t da_lo = MN ? make_sw128_mn_desc(sa_lo) : make_sw128_desc(sa_lo);
    const uint64_t db_hi = MN ? make_sw128_mn_desc(sb_hi) : make_sw128_desc(sb_hi);
    const uint64_t db_lo = MN ? make_sw128_mn_desc(sb_lo) : make_sw128_desc(sb_lo);
    // per K step (16 elements): K-major +32 B inside the swizzle row; MN-major +2 groups of 8 k rows
    constexpr uint64_t kstep = MN ? (uint64_t)((2 * 1024) >> 4) : (uint64_t)((WG_K * 2) >> 4);
#pragma unroll
    for (int k = 0; k < BK / WG_K; ++k) {
        const uint64_t koff = kstep * k;
        wgmma_bf16<BN, MN>(part, da_lo + koff, db_hi + koff, (!chunk_start || k > 0) ? 1u : 0u);
        wgmma_bf16<BN, MN>(part, da_hi + koff, db_lo + koff, 1u);
        wgmma_bf16<BN, MN>(part, da_hi + koff, db_hi + koff, 1u);
    }
}

// K loop of one consumer warpgroup: acc = sum over its k-blocks of the 64 x BN products, promoted every kChunk k-blocks.
// Releases each smem stage (one arrival per warpgroup) once the MMAs reading it have retired.
template <int BN, int MN>
__device__ __forceinline__ void consumer_mainloop(float (&acc)[BN / 2], uint32_t smem_base, uint32_t bar_base, uint32_t a_ofs,
                                                  int num_kb, bool leader, long long* w_full) {
    using Cfg = TileCfg<BN>;
    constexpr int R = BN / 2;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (Cfg::kStages + s); };
    float part[R];
#pragma unroll
    for (int i = 0; i < R; ++i) { acc[i] = 0.f; part[i] = 0.f; }
    for (int kb = 0; kb < num_kb; ++kb) {
        const int s = kb % Cfg::kStages;
        const uint32_t ph = (kb / Cfg::kStages) & 1;
        {
            const long long t0 = w_full ? clock64() : 0;
            mbar_wait(full_bar(s), ph);
            if (w_full) *w_full += clock64() - t0;
        }
        const uint32_t sa_hi = smem_base + s * Cfg::kStageBytes;
        const uint32_t sa_lo = sa_hi + Cfg::kABytes;
        const uint32_t sb_hi = sa_lo + Cfg::kABytes;
        const uint32_t sb_lo = sb_hi + Cfg::kBBytes;
        wgmma_fence();
        mma_stage<BN, MN>(part, sa_hi + a_ofs, sa_lo + a_ofs, sb_hi, sb_lo, (kb % kChunk) == 0);
        wgmma_commit();
        // the other consumer warpgroup's MMAs keep the tensor core busy while this one drains
        wgmma_wait<0>();
        fence_regs(part);
        if (leader) mbar_arrive(empty_bar(s));
        if ((kb % kChunk) == kChunk - 1 || kb == num_kb - 1) {
            // this chunk's partial sum is complete: promote it with round-to-nearest adds
#pragma unroll
            for (int i = 0; i < R; ++i) acc[i] += part[i];
        }
    }
}

template <int BN>
__global__ void __launch_bounds__(NTHREADS, 1)
gemm_bf16x3_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                   const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
                   const GemmParams p) {
    using Cfg = TileCfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_base = smem_base + Cfg::kStages * Cfg::kStageBytes;   // 8-byte aligned
    // barrier layout: full[kStages], empty[kStages]
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (Cfg::kStages + s); };

    const int wg = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 7, 0);      // warp-uniform role index

    // ---- tile coordinates ----
    const int n_tile = blockIdx.x;                 // output column tile
    const int m_tile = blockIdx.y;
    const int zq = (p.mode == 1) ? (int)blockIdx.z : 0;       // mode 1: tap or batch id
    int f0 = 0, n0 = 0, m0 = 0, hb = 0, win = 0;
    const int num_kb = p.num_kb;
    const bool wmap = p.windows > 0;
    if (p.mode == 0) {
        const int mt = wmap ? m_tile % p.win_tiles : m_tile;
        win = wmap ? m_tile / p.win_tiles : 0;
        f0 = mt / p.tiles_per_frame;
        n0 = (mt % p.tiles_per_frame) * BM;
        hb = f0 % p.bmod;
    } else {
        m0 = m_tile * BM;
    }
    const int col0 = n_tile * BN;

    if (threadIdx.x == 0) {
        for (int s = 0; s < Cfg::kStages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (wg == 0) {
        // =============================== TMA producer ===============================
        if (threadIdx.x == 0) {
            long long w_empty = 0;
            for (int kb = 0; kb < num_kb; ++kb) {
                const int s = kb % Cfg::kStages;
                const uint32_t ph = (kb / Cfg::kStages) & 1;
                const long long t0 = p.stats ? clock64() : 0;
                mbar_wait(empty_bar(s), ph ^ 1u);
                if (p.stats) w_empty += clock64() - t0;
                mbar_expect_tx(full_bar(s), Cfg::kStageBytes);
                const uint32_t sa_hi = smem_base + s * Cfg::kStageBytes;
                const uint32_t sa_lo = sa_hi + Cfg::kABytes;
                const uint32_t sb_hi = sa_lo + Cfg::kABytes;
                const uint32_t sb_lo = sb_hi + Cfg::kBBytes;
                if (p.mode == 0) {
                    const int tap = kb / p.kc, c = kb % p.kc;
                    const int dn = tap % p.taps_n - p.taps_n / 2;
                    const int df = tap / p.taps_n - p.taps_f / 2;
                    const int ak = c * BK + hb * p.a_k_bstride;
                    const int af = f0 / p.a_f_div + p.f_start + df;
                    const int bk = c * BK + p.b_k_ofs + hb * p.b_k_bstride;
                    const int bz = tap + hb * p.b_z_bstride;
                    tma_load(wmap, sa_hi, &map_a_hi, full_bar(s), ak, n0 + dn, af, win);
                    tma_load(wmap, sa_lo, &map_a_lo, full_bar(s), ak, n0 + dn, af, win);
                    tma_load_3d(sb_hi, &map_b_hi, full_bar(s), bk, col0, bz);
                    tma_load_3d(sb_lo, &map_b_lo, full_bar(s), bk, col0, bz);
                } else {
                    // K runs over pixels (f, 64-residue block j); operands are MN-major: boxes of
                    // 64 channels x 64 residues, one per 64-wide channel atom.  The tap shift is on the
                    // residue / frame coordinates (row dimensions), out-of-image rows are zero-filled.
                    const int kw = wmap ? kb % p.win_kb : kb;
                    const int wk = wmap ? kb / p.win_kb : 0;
                    const int f = kw / p.kc, j = kw % p.kc;
                    const bool has_taps = p.taps_n * p.taps_f > 1;
                    const int dn = has_taps ? zq % p.taps_n - p.taps_n / 2 : 0;
                    const int df = has_taps ? zq / p.taps_n - p.taps_f / 2 : 0;
                    const int af = f * p.a_f_mul + zq * p.a_z_mul;
                    const int bf = f * p.b_f_mul + zq * p.b_z_mul + p.b_f_add + df;
                    const int bn0 = col0 + zq * p.b_n_zmul;
#pragma unroll
                    for (int a = 0; a < BM / 64; ++a) {
                        tma_load(wmap, sa_hi + a * 8192, &map_a_hi, full_bar(s), m0 + a * 64, j * BK, af, wk);
                        tma_load(wmap, sa_lo + a * 8192, &map_a_lo, full_bar(s), m0 + a * 64, j * BK, af, wk);
                    }
#pragma unroll
                    for (int b = 0; b < BN / 64; ++b) {
                        tma_load(wmap, sb_hi + b * 8192, &map_b_hi, full_bar(s), bn0 + b * 64, j * BK + dn, bf, wk);
                        tma_load(wmap, sb_lo + b * 8192, &map_b_lo, full_bar(s), bn0 + b * 64, j * BK + dn, bf, wk);
                    }
                }
            }
            if (p.stats) {
                const long cta = ((long)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
                p.stats[4 * cta + 2] = w_empty;
                p.stats[4 * cta + 3] = 0;
            }
        }
    } else {
        // =============================== wgmma consumers (warpgroups 1, 2) ===============================
        constexpr int R = BN / 2;                       // accumulator registers per thread (m64nBN)
        const int cw = wg - 1;                          // rows 64 cw .. 64 cw + 63 of the tile
        const int t = threadIdx.x & 127;
        const bool leader = t == 0;
        // rows 64 cw .. of A: K-major 64 rows x 128 B further, MN-major the next 64-wide mn atom -- 8192 B either way
        const uint32_t a_ofs = (uint32_t)cw * 8192u;
        float acc[R];
        long long w_full = 0, t_begin = 0;
        if (p.stats) t_begin = clock64();
        // one K loop per operand layout: the wgmma transpose flags are immediates
        if (p.mode == 1) consumer_mainloop<BN, 1>(acc, smem_base, bar_base, a_ofs, num_kb, leader, p.stats ? &w_full : nullptr);
        else consumer_mainloop<BN, 0>(acc, smem_base, bar_base, a_ofs, num_kb, leader, p.stats ? &w_full : nullptr);
        if (p.stats && cw == 0 && leader) {
            const long cta = ((long)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
            p.stats[4 * cta + 0] = clock64() - t_begin;
            p.stats[4 * cta + 1] = w_full;
        }
        // accumulator layout (m64nBN): register 4 j + 2 h + e holds row 16 warp + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e
        const int warp_in_wg = t >> 5, lane = t & 31;
        const long obase = (p.mode == 1 ? (long)zq * p.out_tap_stride : (long)hb * p.o_col_bstride);
        const bool vec_ok = ((p.ldo & 1) == 0) && ((reinterpret_cast<uintptr_t>(p.out) & 7) == 0) &&
                            (obase % 2 == 0);
        const float* rbase = p.res ? p.res + (p.mode == 0 ? (long)hb * p.o_col_bstride : 0) : nullptr;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = cw * 64 + warp_in_wg * 16 + (lane >> 2) + 8 * h;      // row inside the tile
            long grow;                                                        // global output row
            bool row_ok;
            if (p.mode == 0) {
                const int n = n0 + r;
                grow = ((long)win * p.win_fout + f0 / p.o_f_div) * p.Nr + n;
                row_ok = (n < p.Nr) && (grow < p.out_rows);
            } else {
                grow = m0 + r;
                row_ok = grow < p.out_rows;
            }
            if (!row_ok) continue;
            float* orow = p.out + obase + grow * p.ldo;
            const float* rrow = rbase ? rbase + grow * p.ldr : nullptr;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int gc0 = col0 + 8 * j + 2 * (lane & 3);
                if (gc0 >= p.n_out) break;
                float o[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    float x = acc[4 * j + 2 * h + e] * p.alpha;
                    const int gc = gc0 + e;
                    if (gc < p.n_out) {
                        if (p.bias) x += __ldg(p.bias + gc);
                        if (p.act == 1) x = fmaxf(x, 0.f);
                        else if (p.act == 2) x = x / (1.f + __expf(-x));
                        if (rrow) x += p.beta * __ldg(rrow + gc);
                    }
                    o[e] = x;
                }
                if (vec_ok && gc0 + 2 <= p.n_out) {
                    *reinterpret_cast<float2*>(orow + gc0) = make_float2(o[0], o[1]);
                } else {
                    orow[gc0] = o[0];
                    if (gc0 + 1 < p.n_out) orow[gc0 + 1] = o[1];
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// host side: tensor maps
// ---------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
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

// bf16 tensor with dims d0 (innermost, contiguous), d1, d2 and, when d3 > 0, d3; strides in ELEMENTS for d1, d2, d3.
// The box spans one element of d2 and d3.
int make_map(CUtensorMap* m, const void* base, long d0, long d1, long d2, long s1, long s2, int b0, int b1, int b2,
             long d3 = 0, long s3 = 0) {
    EncodeTiledFn enc = get_encode();
    DFOLD_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled unavailable (driver too old?)");
    DFOLD_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base pointer must be 16-byte aligned");
    DFOLD_REQUIRE((s1 * 2) % 16 == 0 && (s2 * 2) % 16 == 0 && (s3 * 2) % 16 == 0,
                  "TMA strides must be multiples of 16 bytes (s1=%ld s2=%ld s3=%ld)", s1, s2, s3);
    const cuuint32_t rank = d3 > 0 ? 4 : 3;
    cuuint64_t dims[4] = {(cuuint64_t)d0, (cuuint64_t)d1, (cuuint64_t)d2, (cuuint64_t)d3};
    cuuint64_t strides[3] = {(cuuint64_t)s1 * 2, (cuuint64_t)s2 * 2, (cuuint64_t)s3 * 2};
    cuuint32_t box[4] = {(cuuint32_t)b0, (cuuint32_t)b1, (cuuint32_t)b2, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(base), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    DFOLD_REQUIRE(r == CUDA_SUCCESS,
                  "cuTensorMapEncodeTiled failed (%d) dims=(%ld,%ld,%ld,%ld) strides=(%ld,%ld,%ld) box=(%d,%d,%d)",
                  (int)r, d0, d1, d2, d3, s1, s2, s3, b0, b1, b2);
    return 0;
}

long long* g_stats = nullptr;      // set by dfold_debug_gemm_stats

template <int BN>
int launch(const CUtensorMap* maps, const GemmParams& p_in, dim3 grid, cudaStream_t st) {
    using Cfg = TileCfg<BN>;
    GemmParams p = p_in;
    p.stats = g_stats;
    static SmemCfg cfg;
    if (ensure_dyn_smem(gemm_bf16x3_kernel<BN>, Cfg::kSmemBytes, cfg, "gemm_bf16x3_kernel")) return 1;
    gemm_bf16x3_kernel<BN><<<grid, NTHREADS, Cfg::kSmemBytes, st>>>(maps[0], maps[1], maps[2], maps[3], p);
    return check_launch("gemm_bf16x3_kernel");
}

int sm_count() {
    static int n[64] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
    dev &= 63;
    if (n[dev] == 0) {
        if (cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n[dev] <= 0) n[dev] = 132;
    }
    return n[dev];
}

void default_batching(GemmParams& p) {
    p.bmod = 1; p.a_f_div = 1; p.a_k_bstride = 0; p.b_k_ofs = 0; p.b_k_bstride = 0; p.b_z_bstride = 0;
    p.o_f_div = 1; p.o_col_bstride = 0; p.f_start = 0; p.b_f_add = 0;
    p.a_f_mul = 1; p.a_z_mul = 0; p.b_f_mul = 1; p.b_z_mul = 0; p.b_n_zmul = 0;
    p.windows = 0; p.win_tiles = 0; p.win_fout = 0; p.win_kb = 0;
}


// Tile width: every CTA owns one SM (up to 227 KB of shared memory; the 128-wide ring takes 192 KB), so the launch runs
// in ceil(tiles / SMs) waves, here taken to last in proportion to BN.  Pick the width with the smallest waves x BN
// (ties -> the wider tile, which re-reads the A operand less).  A 64-wide tile in fact takes ~0.6 of a 128-wide one's
// time, so the convolutions choose their width from that measured cost through the *_bn entry points (DESIGN.md §4).  `row_tiles` = 128-row tiles x batches / taps in the other
// grid dimensions.  BN stops at 128: a 64 x BN wgmma tile per consumer warpgroup holds BN / 2 accumulator registers per
// thread twice over (tensor-core partial sum + promoted sum), and BN = 256 would need 256 of them.
int pick_bn(long n_out, long row_tiles) {
    if (n_out <= 64) return 64;
    const long sms = sm_count();
    const long t128 = cdiv(n_out, 128) * row_tiles, t64 = cdiv(n_out, 64) * row_tiles;
    const long c128 = cdiv(t128, sms) * 128, c64 = cdiv(t64, sms) * 64;
    return (c64 < c128) ? 64 : 128;
}

}  // namespace
}  // namespace dfold

using namespace dfold;

// ---------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------
// Development aid: when `buf` (device, 4 x int64 per CTA of the next launches) is non-null every GEMM launch records, per
// CTA, the cycles of its first consumer warpgroup's mainloop and the cycles the consumers / the producer spent waiting on barriers.
extern "C" int dfold_debug_gemm_stats(long long* buf) {
    g_stats = buf;
    return 0;
}

namespace dfold {
namespace {

// dfold_gemm_bf16x3 on tiles `bn` wide.  `name`: the calling entry point, for error messages.  W > 0: W stacked windows
// of F frames each (dfold_gemm_bf16x3_windows); W = 0: one image of F frames on 3-D maps.
int gemm_kmajor(const char* name, const uint16_t* a_hi, const uint16_t* a_lo, long W, long F, long F_out, int f_start,
                long Nr, long K, long lda, const uint16_t* b_hi, const uint16_t* b_lo, long n_out, long ldb, int taps_f,
                int taps_n, float* out, long ldo, const float* bias, const float* residual, long ldr,
                float alpha, float beta, int act, int bn, void* stream) {
    DFOLD_REQUIRE(F > 0 && F_out > 0 && Nr > 0 && K > 0 && n_out > 0 && W >= 0, "%s: empty problem", name);
    DFOLD_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "%s: lda/ldb must be multiples of 8 (got %ld, %ld)", name, lda, ldb);
    DFOLD_REQUIRE(taps_f >= 1 && taps_n >= 1 && (taps_f & 1) && (taps_n & 1), "%s: tap grid must be odd", name);
    DFOLD_REQUIRE(bn == 64 || bn == 128, "%s: tile width must be 64 or 128 (got %d)", name, bn);
    const long row_tiles = F_out * cdiv(Nr, BM);
    DFOLD_REQUIRE((W > 0 ? W : 1) * row_tiles <= 65535, "%s: too many row tiles (%ld)", name, (W > 0 ? W : 1) * row_tiles);
    CUtensorMap maps[4];
    // A: dims (K, Nr, F [, W])   B: dims (K, n_out, taps)
    if (make_map(&maps[0], a_hi, K, Nr, F, lda, Nr * lda, BK, BM, 1, W, F * Nr * lda)) return 1;
    if (make_map(&maps[1], a_lo, K, Nr, F, lda, Nr * lda, BK, BM, 1, W, F * Nr * lda)) return 1;
    const long taps = (long)taps_f * taps_n;
    if (make_map(&maps[2], b_hi, K, n_out, taps, ldb, n_out * ldb, BK, bn, 1)) return 1;
    if (make_map(&maps[3], b_lo, K, n_out, taps, ldb, n_out * ldb, BK, bn, 1)) return 1;
    GemmParams p{};
    p.mode = 0;
    p.kc = (int)cdiv(K, BK);
    p.num_kb = (int)(taps * p.kc);
    p.taps_n = taps_n; p.taps_f = taps_f;
    p.tiles_per_frame = (int)cdiv(Nr, BM);
    p.Nr = (int)Nr;
    p.out_rows = (W > 0 ? W : 1) * F_out * Nr;
    p.n_out = (int)n_out;
    p.out = out; p.ldo = ldo; p.out_tap_stride = 0;
    p.bias = bias; p.res = residual; p.ldr = ldr;
    p.alpha = alpha; p.beta = beta; p.act = act;
    default_batching(p);
    p.f_start = f_start;
    p.windows = (int)W; p.win_tiles = (int)row_tiles; p.win_fout = (int)F_out;
    cudaStream_t st = as_stream(stream);
    // Every output element is produced by one CTA in a fixed k order (no split-K with atomics): the result is the same
    // from run to run, and the same at either tile width.  A row tile lies in one frame of one window.
    dim3 grid((unsigned)cdiv(n_out, bn), (unsigned)((W > 0 ? W : 1) * row_tiles), 1);
    if (bn == 128) return launch<128>(maps, p, grid, st);
    return launch<64>(maps, p, grid, st);
}

// dfold_gemm_wgrad_bf16x3 on tiles `bn` wide.  W > 0: the reduction runs over the pixels of W stacked windows, window
// by window (dfold_gemm_wgrad_bf16x3_windows); W = 0: one image on 3-D maps.
int gemm_wgrad(const char* name, const uint16_t* a_hi, const uint16_t* a_lo, long M, long lda,
               const uint16_t* b_hi, const uint16_t* b_lo, long Nn, long ldb,
               long W, long F, long Fb, int b_f_add, long Nr, int taps_f, int taps_n,
               float* out, long ldo, float alpha, int bn, void* stream) {
    DFOLD_REQUIRE(M > 0 && Nn > 0 && F > 0 && Fb > 0 && Nr > 0 && W >= 0, "%s: empty problem", name);
    DFOLD_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "%s: lda/ldb must be multiples of 8 (got %ld, %ld)", name, lda, ldb);
    DFOLD_REQUIRE(bn == 64 || bn == 128, "%s: tile width must be 64 or 128 (got %d)", name, bn);
    CUtensorMap maps[4];
    // dims (channel, residue, frame [, window]); boxes of 64 channels x 64 residues
    if (make_map(&maps[0], a_hi, M, Nr, F, lda, Nr * lda, 64, BK, 1, W, F * Nr * lda)) return 1;
    if (make_map(&maps[1], a_lo, M, Nr, F, lda, Nr * lda, 64, BK, 1, W, F * Nr * lda)) return 1;
    if (make_map(&maps[2], b_hi, Nn, Nr, Fb, ldb, Nr * ldb, 64, BK, 1, W, Fb * Nr * ldb)) return 1;
    if (make_map(&maps[3], b_lo, Nn, Nr, Fb, ldb, Nr * ldb, 64, BK, 1, W, Fb * Nr * ldb)) return 1;
    GemmParams p{};
    p.mode = 1;
    p.kc = (int)cdiv(Nr, BK);
    p.num_kb = (int)((W > 0 ? W : 1) * F * p.kc);
    p.taps_n = taps_n; p.taps_f = taps_f;
    p.tiles_per_frame = 1; p.Nr = (int)Nr;
    p.out_rows = M; p.n_out = (int)Nn;
    p.out = out; p.ldo = ldo; p.out_tap_stride = M * ldo;
    p.bias = nullptr; p.res = nullptr; p.ldr = 0;
    p.alpha = alpha; p.beta = 0.f; p.act = 0;
    default_batching(p);
    p.b_f_add = b_f_add;
    p.windows = (int)W; p.win_kb = (int)(F * p.kc);
    dim3 grid((unsigned)cdiv(Nn, bn), (unsigned)cdiv(M, BM), (unsigned)(taps_f * taps_n));
    cudaStream_t st = as_stream(stream);
    if (bn == 128) return launch<128>(maps, p, grid, st);
    return launch<64>(maps, p, grid, st);
}

}  // namespace
}  // namespace dfold

extern "C" int dfold_gemm_bf16x3(
    const uint16_t* a_hi, const uint16_t* a_lo, long F, long F_out, int f_start, long Nr, long K, long lda,
    const uint16_t* b_hi, const uint16_t* b_lo, long n_out, long ldb, int taps_f, int taps_n,
    float* out, long ldo, const float* bias, const float* residual, long ldr,
    float alpha, float beta, int act, void* stream) {
    return gemm_kmajor("dfold_gemm_bf16x3", a_hi, a_lo, 0, F, F_out, f_start, Nr, K, lda, b_hi, b_lo, n_out, ldb, taps_f,
                       taps_n, out, ldo, bias, residual, ldr, alpha, beta, act, pick_bn(n_out, F_out * cdiv(Nr, BM)), stream);
}

// dfold_gemm_bf16x3 on tiles `bn` (64 or 128) wide, for callers that weigh the widths themselves.
extern "C" int dfold_gemm_bf16x3_bn(
    const uint16_t* a_hi, const uint16_t* a_lo, long F, long F_out, int f_start, long Nr, long K, long lda,
    const uint16_t* b_hi, const uint16_t* b_lo, long n_out, long ldb, int taps_f, int taps_n,
    float* out, long ldo, const float* bias, const float* residual, long ldr,
    float alpha, float beta, int act, int bn, void* stream) {
    return gemm_kmajor("dfold_gemm_bf16x3_bn", a_hi, a_lo, 0, F, F_out, f_start, Nr, K, lda, b_hi, b_lo, n_out, ldb, taps_f,
                       taps_n, out, ldo, bias, residual, ldr, alpha, beta, act, bn, stream);
}

// out[tap][m][n] = alpha * sum_{f, j} A[f][j][m] * B[f + df(tap)][j + dn(tap)][n]      (weight gradient; K = pixels)
// A planes [F][Nr][lda] (e.g. the gated output gradient, m = output channel), B planes [Fb][Nr][ldb] (the layer input,
// n = input channel, frame f of A pairs with frame f + b_f_add of B: cropped convolutions): the SAME pixel-major
// planes the forward / data-gradient GEMMs use, read MN-major.
extern "C" int dfold_gemm_wgrad_bf16x3(
    const uint16_t* a_hi, const uint16_t* a_lo, long M, long lda,
    const uint16_t* b_hi, const uint16_t* b_lo, long Nn, long ldb,
    long F, long Fb, int b_f_add, long Nr, int taps_f, int taps_n,
    float* out, long ldo, float alpha, void* stream) {
    return gemm_wgrad("dfold_gemm_wgrad_bf16x3", a_hi, a_lo, M, lda, b_hi, b_lo, Nn, ldb, 0, F, Fb, b_f_add, Nr, taps_f, taps_n,
                      out, ldo, alpha, pick_bn(Nn, cdiv(M, BM) * taps_f * taps_n), stream);
}

// dfold_gemm_wgrad_bf16x3 on tiles `bn` (64 or 128) wide.
extern "C" int dfold_gemm_wgrad_bf16x3_bn(
    const uint16_t* a_hi, const uint16_t* a_lo, long M, long lda,
    const uint16_t* b_hi, const uint16_t* b_lo, long Nn, long ldb,
    long F, long Fb, int b_f_add, long Nr, int taps_f, int taps_n,
    float* out, long ldo, float alpha, int bn, void* stream) {
    return gemm_wgrad("dfold_gemm_wgrad_bf16x3_bn", a_hi, a_lo, M, lda, b_hi, b_lo, Nn, ldb, 0, F, Fb, b_f_add, Nr, taps_f,
                      taps_n, out, ldo, alpha, bn, stream);
}

// dfold_gemm_bf16x3_bn over W >= 1 stacked windows: A planes [W][F][Nr][lda], output / residual rows (w * F_out + f) * Nr + n.
// Each window is convolved on its own: the frame halo is zero-filled at every window's edge.
extern "C" int dfold_gemm_bf16x3_windows(
    const uint16_t* a_hi, const uint16_t* a_lo, long W, long F, long F_out, int f_start, long Nr, long K, long lda,
    const uint16_t* b_hi, const uint16_t* b_lo, long n_out, long ldb, int taps_f, int taps_n,
    float* out, long ldo, const float* bias, const float* residual, long ldr,
    float alpha, float beta, int act, int bn, void* stream) {
    DFOLD_REQUIRE(W >= 1, "dfold_gemm_bf16x3_windows: need at least one window (got %ld)", W);
    return gemm_kmajor("dfold_gemm_bf16x3_windows", a_hi, a_lo, W, F, F_out, f_start, Nr, K, lda, b_hi, b_lo, n_out, ldb,
                       taps_f, taps_n, out, ldo, bias, residual, ldr, alpha, beta, act, bn, stream);
}

// dfold_gemm_wgrad_bf16x3_bn summed over W >= 1 stacked windows: A planes [W][F][Nr][lda], B planes [W][Fb][Nr][ldb];
// frame f of A's window w pairs with frame f + b_f_add of B's window w, and taps never reach into another window.
extern "C" int dfold_gemm_wgrad_bf16x3_windows(
    const uint16_t* a_hi, const uint16_t* a_lo, long M, long lda,
    const uint16_t* b_hi, const uint16_t* b_lo, long Nn, long ldb,
    long W, long F, long Fb, int b_f_add, long Nr, int taps_f, int taps_n,
    float* out, long ldo, float alpha, int bn, void* stream) {
    DFOLD_REQUIRE(W >= 1, "dfold_gemm_wgrad_bf16x3_windows: need at least one window (got %ld)", W);
    return gemm_wgrad("dfold_gemm_wgrad_bf16x3_windows", a_hi, a_lo, M, lda, b_hi, b_lo, Nn, ldb, W, F, Fb, b_f_add, Nr,
                      taps_f, taps_n, out, ldo, alpha, bn, stream);
}

// Batched K-major GEMM (no taps): for every row tile of "frame" b in [0, n_batches), hb = b % bmod:
//   out[(b / o_f_div) * Nr + n, hb * o_col_bstride + c] = alpha * sum_k A[b / a_f_div][n][hb * a_k_bstride + k]
//                                                                    * B[hb * b_z_bstride][c][b_k_ofs + hb * b_k_bstride + k]
// A planes: [a_frames][Nr][lda]; B planes: [b_z][b_rows][ldb].
extern "C" int dfold_gemm_bf16x3_batched(
    const uint16_t* a_hi, const uint16_t* a_lo, long a_frames, long Nr, long a_cols, long lda,
    long n_batches, int bmod, int a_f_div, long a_k_bstride, long K,
    const uint16_t* b_hi, const uint16_t* b_lo, long b_z, long b_rows, long b_cols, long ldb,
    long b_k_ofs, long b_k_bstride, int b_z_bstride, long n_out,
    float* out, long ldo, long out_rows, int o_f_div, long o_col_bstride, float alpha, void* stream) {
    DFOLD_REQUIRE(n_batches > 0 && Nr > 0 && K > 0 && n_out > 0 && bmod >= 1, "dfold_gemm_bf16x3_batched: empty problem");
    DFOLD_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "dfold_gemm_bf16x3_batched: lda/ldb must be multiples of 8");
    DFOLD_REQUIRE(a_k_bstride % 8 == 0 && b_k_ofs % 8 == 0 && b_k_bstride % 8 == 0,
                  "dfold_gemm_bf16x3_batched: K offsets must be multiples of 8 elements (TMA 16-byte alignment)");
    // K tail: the A / B boxes may run past [k_ofs, k_ofs + K) into the neighbouring batch slice; require K % 64 == 0
    const bool k_sliced = a_k_bstride != 0 || b_k_ofs != 0 || b_k_bstride != 0;
    DFOLD_REQUIRE(K % BK == 0 || !k_sliced,
                  "dfold_gemm_bf16x3_batched: K must be a multiple of 64 when it is a slice of a wider row");
    // Unsliced, the reduction covers columns [0, K): the maps end there, so a K tail reads the out-of-bounds zero fill
    // and not the columns of rows that are wider than K.
    const long a_k_end = k_sliced ? a_cols : (a_cols < K ? a_cols : K);
    const long b_k_end = k_sliced ? b_cols : (b_cols < K ? b_cols : K);
    const int bn = pick_bn(n_out, n_batches * cdiv(Nr, BM));
    CUtensorMap maps[4];
    if (make_map(&maps[0], a_hi, a_k_end, Nr, a_frames, lda, Nr * lda, BK, BM, 1)) return 1;
    if (make_map(&maps[1], a_lo, a_k_end, Nr, a_frames, lda, Nr * lda, BK, BM, 1)) return 1;
    if (make_map(&maps[2], b_hi, b_k_end, b_rows, b_z, ldb, b_rows * ldb, BK, bn, 1)) return 1;
    if (make_map(&maps[3], b_lo, b_k_end, b_rows, b_z, ldb, b_rows * ldb, BK, bn, 1)) return 1;
    GemmParams p{};
    p.mode = 0;
    p.kc = (int)cdiv(K, BK);
    p.num_kb = p.kc;
    p.taps_n = 1; p.taps_f = 1;
    p.tiles_per_frame = (int)cdiv(Nr, BM);
    p.Nr = (int)Nr;
    p.out_rows = out_rows;
    p.n_out = (int)n_out;
    p.out = out; p.ldo = ldo; p.out_tap_stride = 0;
    p.bias = nullptr; p.res = nullptr; p.ldr = 0;
    p.alpha = alpha; p.beta = 0.f; p.act = 0;
    default_batching(p);
    p.bmod = bmod; p.a_f_div = a_f_div; p.a_k_bstride = (int)a_k_bstride;
    p.b_k_ofs = (int)b_k_ofs; p.b_k_bstride = (int)b_k_bstride; p.b_z_bstride = b_z_bstride;
    p.o_f_div = o_f_div; p.o_col_bstride = o_col_bstride;
    dim3 grid((unsigned)cdiv(n_out, bn), (unsigned)(n_batches * p.tiles_per_frame), 1);
    cudaStream_t st = as_stream(stream);
    if (bn == 128) return launch<128>(maps, p, grid, st);
    return launch<64>(maps, p, grid, st);
}

// Batched MN-major GEMM (K = rows):  for z in [0, zcount)
//   out[z][m][n] = alpha * sum_{f < Fk} sum_j A[f * a_f_mul + z * a_z_mul][j][m] * B[f * b_f_mul + z * b_z_mul][j][z * b_n_zmul + n]
// A planes: dims (M, a_mid, a_outer) with element strides (lda, a_ostride); B likewise.  K loop: Fk outer x ceil(Nr/64) blocks.
extern "C" int dfold_gemm_wgrad_bf16x3_batched(
    const uint16_t* a_hi, const uint16_t* a_lo, long M, long a_mid, long a_outer, long lda, long a_ostride,
    const uint16_t* b_hi, const uint16_t* b_lo, long b_cols, long b_mid, long b_outer, long ldb, long b_ostride,
    long Nn, long Fk, long Nr, int zcount, int a_f_mul, int a_z_mul, int b_f_mul, int b_z_mul, long b_n_zmul,
    float* out, long ldo, long out_z_stride, float alpha, void* stream) {
    DFOLD_REQUIRE(M > 0 && Nn > 0 && Fk > 0 && Nr > 0 && zcount > 0, "dfold_gemm_wgrad_bf16x3_batched: empty problem");
    DFOLD_REQUIRE(lda % 8 == 0 && ldb % 8 == 0 && a_ostride % 8 == 0 && b_ostride % 8 == 0 && b_n_zmul % 8 == 0,
                  "dfold_gemm_wgrad_bf16x3_batched: strides / offsets must be multiples of 8 elements");
    const int bn = pick_bn(Nn, cdiv(M, BM) * zcount);
    CUtensorMap maps[4];
    if (make_map(&maps[0], a_hi, M, a_mid, a_outer, lda, a_ostride, 64, BK, 1)) return 1;
    if (make_map(&maps[1], a_lo, M, a_mid, a_outer, lda, a_ostride, 64, BK, 1)) return 1;
    if (make_map(&maps[2], b_hi, b_cols, b_mid, b_outer, ldb, b_ostride, 64, BK, 1)) return 1;
    if (make_map(&maps[3], b_lo, b_cols, b_mid, b_outer, ldb, b_ostride, 64, BK, 1)) return 1;
    GemmParams p{};
    p.mode = 1;
    p.kc = (int)cdiv(Nr, BK);
    p.num_kb = (int)(Fk * p.kc);
    p.taps_n = 1; p.taps_f = 1;
    p.tiles_per_frame = 1; p.Nr = (int)Nr;
    p.out_rows = M; p.n_out = (int)Nn;
    p.out = out; p.ldo = ldo; p.out_tap_stride = out_z_stride;
    p.bias = nullptr; p.res = nullptr; p.ldr = 0;
    p.alpha = alpha; p.beta = 0.f; p.act = 0;
    default_batching(p);
    p.a_f_mul = a_f_mul; p.a_z_mul = a_z_mul; p.b_f_mul = b_f_mul; p.b_z_mul = b_z_mul; p.b_n_zmul = (int)b_n_zmul;
    DFOLD_REQUIRE(zcount <= 65535, "dfold_gemm_wgrad_bf16x3_batched: too many z blocks");
    dim3 grid((unsigned)cdiv(Nn, bn), (unsigned)cdiv(M, BM), (unsigned)zcount);
    cudaStream_t st = as_stream(stream);
    if (bn == 128) return launch<128>(maps, p, grid, st);
    return launch<64>(maps, p, grid, st);
}
