// CUDA-core kernels of the dfold_b200 library: operand preparation for the split-bf16 GEMM, a generic strided
// fp32 GEMM for shapes the tensor-core tile cannot take, whole-tensor and per-row layer norms.
#include <stdarg.h>
#include <string.h>
#include "common.cuh"

namespace dfold {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return 1;
    }
    return 0;
}

namespace {

__device__ __forceinline__ uint32_t split_pack(float x) {
    // hi = bf16(x), lo = bf16(x - hi); packed (hi << 16) | lo
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
    return ((uint32_t)__bfloat16_as_ushort(h) << 16) | (uint32_t)__bfloat16_as_ushort(l);
}

// The ReLU gate of a layer at element i: gate > 0, or (gate - gate_sub) > 0 for a residual layer whose gate is its output
// minus the residual.  The fp32 subtraction rounds as torch's would, so the gate opens on exactly the same elements.
__device__ __forceinline__ bool gate_open(const float* __restrict__ gate, const float* __restrict__ gate_sub, long i) {
    return (gate_sub ? gate[i] - gate_sub[i] : gate[i]) > 0.f;
}

// x[R, C] (row stride ld) -> hi/lo [R, ldo] and optionally transposed hi_t/lo_t [C, ldt].
// Optional: relu on the input, a gate (x *= gate_open).  The column sums of the (gated) input come from colsum_kernel.
__global__ void split2d_kernel(const float* __restrict__ x, long R, long C, long ld, int pre_relu,
                               const float* __restrict__ gate, const float* __restrict__ gate_sub, long ldg,
                               uint16_t* __restrict__ hi, uint16_t* __restrict__ lo, long ldo, long cpad,
                               uint16_t* __restrict__ hit, uint16_t* __restrict__ lot, long ldt, long rpad) {
    __shared__ uint32_t tile[32][33];
    const long r0 = (long)blockIdx.y * 32, c0 = (long)blockIdx.x * 32;
    const int tx = threadIdx.x, ty = threadIdx.y;       // 32 x 8
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long r = r0 + ty + i * 8, c = c0 + tx;
        float v = 0.f;
        if (r < R && c < C) {
            v = x[r * ld + c];
            if (pre_relu) v = fmaxf(v, 0.f);
            if (gate) v = gate_open(gate, gate_sub, r * ldg + c) ? v : 0.f;
        }
        const uint32_t pk = split_pack(v);
        tile[ty + i * 8][tx] = pk;
        if (hi && r < R && c < cpad) {      // columns in [C, cpad) are written as zero padding
            hi[r * ldo + c] = (uint16_t)(pk >> 16);
            lo[r * ldo + c] = (uint16_t)(pk & 0xffffu);
        }
    }
    __syncthreads();
    if (hit) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const long c = c0 + ty + i * 8, r = r0 + tx;   // transposed: row index = original column
            if (c < C && r < rpad) {
                const uint32_t pk = (r < R) ? tile[tx][ty + i * 8] : 0u;
                hit[c * ldt + r] = (uint16_t)(pk >> 16);
                lot[c * ldt + r] = (uint16_t)(pk & 0xffffu);
            }
        }
    }
}

// Row-major fast path of split2d (no transposed planes, no column sums, 16-byte aligned rows): one thread = four consecutive
// columns, float4 in, 8 bytes of each plane out.
__global__ void __launch_bounds__(256) split2d_vec_kernel(const float* __restrict__ x, long R, long C, long ld, int pre_relu,
                                                          const float* __restrict__ gate, const float* __restrict__ gate_sub,
                                                          long ldg, uint16_t* __restrict__ hi,
                                                          uint16_t* __restrict__ lo, long ldo, long c4n) {
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= R * c4n) return;
    const long r = idx / c4n, c = (idx % c4n) * 4;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (c + 4 <= C) {
        const float4 t = *reinterpret_cast<const float4*>(x + r * ld + c);
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
        if (gate) {
            float4 g = *reinterpret_cast<const float4*>(gate + r * ldg + c);
            if (gate_sub) {
                const float4 s = *reinterpret_cast<const float4*>(gate_sub + r * ldg + c);
                g.x -= s.x; g.y -= s.y; g.z -= s.z; g.w -= s.w;
            }
            v[0] = g.x > 0.f ? v[0] : 0.f; v[1] = g.y > 0.f ? v[1] : 0.f; v[2] = g.z > 0.f ? v[2] : 0.f; v[3] = g.w > 0.f ? v[3] : 0.f;
        }
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (c + k < C) {
                v[k] = x[r * ld + c + k];
                if (gate) v[k] = gate_open(gate, gate_sub, r * ldg + c + k) ? v[k] : 0.f;
            }
    }
    if (pre_relu) {                     // relu and the gate commute: relu(gate ? v : 0) == gate ? relu(v) : 0
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = fmaxf(v[k], 0.f);
    }
    uint32_t pk[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) pk[k] = split_pack(v[k]);
    *reinterpret_cast<uint2*>(hi + r * ldo + c) = make_uint2((pk[0] >> 16) | (pk[1] & 0xffff0000u), (pk[2] >> 16) | (pk[3] & 0xffff0000u));
    *reinterpret_cast<uint2*>(lo + r * ldo + c) = make_uint2((pk[0] & 0xffffu) | (pk[1] << 16), (pk[2] & 0xffffu) | (pk[3] << 16));
}

// conv weight w[O][I][T] (T = taps, contiguous) ->
//   fwd planes   [T][O][ldi]   (K = I contiguous)
//   dgrad planes [T][I][ldo_]  (K = O contiguous), tap index flipped (T-1-t)
// One CTA per 32 x 32 (o, i) tile: the tile is read with 32 contiguous runs of 32*T floats and both plane sets are
// written in 64-byte runs (i-contiguous for the forward planes, o-contiguous for the dgrad planes).
__global__ void __launch_bounds__(256) conv_weight_prep_kernel(const float* __restrict__ w, int O, int I, int T,
                                        uint16_t* __restrict__ f_hi, uint16_t* __restrict__ f_lo, long ldi,
                                        uint16_t* __restrict__ d_hi, uint16_t* __restrict__ d_lo, long ldo_) {
    extern __shared__ uint32_t sm[];                  // [32 o][32 i][T]  (+1 padding per o row)
    const int o0 = blockIdx.y * 32, i0 = blockIdx.x * 32;
    const int no = min(32, O - o0), ni = min(32, I - i0);
    const int row = 32 * T + 1;
    for (int oo = 0; oo < no; ++oo) {
        const float* src = w + ((long)(o0 + oo) * I + i0) * T;
        for (int e = threadIdx.x; e < ni * T; e += blockDim.x) sm[oo * row + e] = split_pack(src[e]);
    }
    __syncthreads();
    if (no == 32 && ni == 32 && (ldi & 3) == 0 && (d_hi == nullptr || (ldo_ & 3) == 0)) {
        // full tile: 8-byte stores (4 bf16 of one plane), 8 lanes per 64-byte row
        for (int e = threadIdx.x; e < T * 32 * 8; e += blockDim.x) {
            const int q = e & 7, oo = (e >> 3) & 31, t = e >> 8;
            uint32_t pk[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) pk[c] = sm[oo * row + (4 * q + c) * T + t];
            const long fo = ((long)t * O + o0 + oo) * ldi + i0 + 4 * q;
            *reinterpret_cast<uint2*>(f_hi + fo) = make_uint2((pk[0] >> 16) | (pk[1] & 0xffff0000u), (pk[2] >> 16) | (pk[3] & 0xffff0000u));
            *reinterpret_cast<uint2*>(f_lo + fo) = make_uint2((pk[0] & 0xffffu) | (pk[1] << 16), (pk[2] & 0xffffu) | (pk[3] << 16));
        }
        if (d_hi) {
            for (int e = threadIdx.x; e < T * 32 * 8; e += blockDim.x) {
                const int q = e & 7, ii = (e >> 3) & 31, t = e >> 8;
                uint32_t pk[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) pk[c] = sm[(4 * q + c) * row + ii * T + t];
                const long dofs = ((long)(T - 1 - t) * I + i0 + ii) * ldo_ + o0 + 4 * q;
                *reinterpret_cast<uint2*>(d_hi + dofs) = make_uint2((pk[0] >> 16) | (pk[1] & 0xffff0000u), (pk[2] >> 16) | (pk[3] & 0xffff0000u));
                *reinterpret_cast<uint2*>(d_lo + dofs) = make_uint2((pk[0] & 0xffffu) | (pk[1] << 16), (pk[2] & 0xffffu) | (pk[3] << 16));
            }
        }
        return;
    }
    // forward planes: (t, o) rows, i contiguous
    for (int e = threadIdx.x; e < T * 32 * 32; e += blockDim.x) {
        const int ii = e & 31, oo = (e >> 5) & 31, t = e >> 10;
        if (ii < ni && oo < no) {
            const uint32_t pk = sm[oo * row + ii * T + t];
            const long fo = ((long)t * O + o0 + oo) * ldi + i0 + ii;
            f_hi[fo] = (uint16_t)(pk >> 16);
            f_lo[fo] = (uint16_t)(pk & 0xffffu);
        }
    }
    if (d_hi) {
        // dgrad planes: (t', i) rows, o contiguous
        for (int e = threadIdx.x; e < T * 32 * 32; e += blockDim.x) {
            const int oo = e & 31, ii = (e >> 5) & 31, t = e >> 10;
            if (ii < ni && oo < no) {
                const uint32_t pk = sm[oo * row + ii * T + t];
                const long dofs = ((long)(T - 1 - t) * I + i0 + ii) * ldo_ + o0 + oo;
                d_hi[dofs] = (uint16_t)(pk >> 16);
                d_lo[dofs] = (uint16_t)(pk & 0xffffu);
            }
        }
    }
}

// g[T][O][I] -> out[O][I][T]   (weight-gradient layout back to the parameter's [C_out, C_in, 5, 5])
__global__ void taps_to_param_kernel(const float* __restrict__ g, int O, int I, int T, float* __restrict__ out, int accumulate) {
    extern __shared__ float smf[];                    // [T][65]
    const int o = blockIdx.y;
    const int i0 = blockIdx.x * 64;
    const int ni = min(64, I - i0);
    for (int e = threadIdx.x; e < T * 64; e += blockDim.x) {
        const int t = e / 64, ii = e % 64;
        if (ii < ni) smf[t * 65 + ii] = g[((long)t * O + o) * I + i0 + ii];
    }
    __syncthreads();
    float* dst = out + ((long)o * I + i0) * T;
    for (int e = threadIdx.x; e < ni * T; e += blockDim.x) {
        const int ii = e / T, t = e % T;
        dst[e] = (accumulate ? dst[e] : 0.f) + smf[t * 65 + ii];
    }
}

// ---------------------------------------------------------------------------------------------------
// generic strided fp32 GEMM:  C[b][m][n] = act(alpha * sum_k A[b][m][k] * B[b][n][k] + bias[n]) + beta * R[b][m][n]
// ---------------------------------------------------------------------------------------------------
struct SgemmParams {
    const float* A; long a_rs, a_cs, a_bs, a_bs2;
    const float* B; long b_rs, b_cs, b_bs, b_bs2;
    float* C; long c_rs, c_cs, c_bs, c_bs2;
    const float* R; long r_rs, r_cs, r_bs, r_bs2;
    const float* bias;
    int nb2;
    int ksplit;          // > 1: blockIdx.z also enumerates K chunks; partial sums are atomically added to a zeroed C
    int M, N, K;
    float alpha, beta;
    int act, pre_relu;
};

__global__ void __launch_bounds__(256) sgemm_kernel(const SgemmParams p) {
    __shared__ float As[16][65];
    __shared__ float Bs[16][65];
    const int zb = blockIdx.z / p.ksplit, ks = blockIdx.z % p.ksplit;
    const int b = zb / p.nb2, b2 = zb % p.nb2;
    const int kchunk = ((p.K + p.ksplit - 1) / p.ksplit + 15) / 16 * 16;
    const int kbeg = ks * kchunk, kend = min(p.K, kbeg + kchunk);
    const float* A = p.A + (long)b * p.a_bs + (long)b2 * p.a_bs2;
    const float* B = p.B + (long)b * p.b_bs + (long)b2 * p.b_bs2;
    const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;           // 16 x 16 threads, 4x4 outputs each
    float acc[4][4] = {};
    for (int k0 = kbeg; k0 < kend; k0 += 16) {
#pragma unroll
        for (int e = tid; e < 64 * 16; e += 256) {
            // choose the faster-varying index to follow the contiguous direction of the operand
            int mm, kk;
            if (p.a_cs == 1) { kk = e & 15; mm = e >> 4; } else { mm = e & 63; kk = e >> 6; }
            float v = 0.f;
            if (m0 + mm < p.M && k0 + kk < kend) {
                v = A[(long)(m0 + mm) * p.a_rs + (long)(k0 + kk) * p.a_cs];
                if (p.pre_relu) v = fmaxf(v, 0.f);
            }
            As[kk][mm] = v;
            int nn, kb;
            if (p.b_cs == 1) { kb = e & 15; nn = e >> 4; } else { nn = e & 63; kb = e >> 6; }
            float u = 0.f;
            if (n0 + nn < p.N && k0 + kb < kend) u = B[(long)(n0 + nn) * p.b_rs + (long)(k0 + kb) * p.b_cs];
            Bs[kb][nn] = u;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < 16; ++kk) {
            float a[4], bv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) bv[j] = Bs[kk][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
    float* C = p.C + (long)b * p.c_bs + (long)b2 * p.c_bs2;
    const float* R = p.R ? p.R + (long)b * p.r_bs + (long)b2 * p.r_bs2 : nullptr;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= p.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= p.N) continue;
            float x = acc[i][j] * p.alpha;
            if (p.ksplit > 1) {
                atomicAdd(&C[(long)m * p.c_rs + (long)n * p.c_cs], x);
                continue;
            }
            if (p.bias) x += p.bias[n];
            if (p.act == 1) x = fmaxf(x, 0.f);
            else if (p.act == 2) x = x / (1.f + expf(-x));
            if (R) x += p.beta * R[(long)m * p.r_rs + (long)n * p.r_cs];
            C[(long)m * p.c_rs + (long)n * p.c_cs] = x;
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// whole-tensor layer norm (MyLayerNorm, reference ipa_pytorch_dynamic.py:709-724)
// ---------------------------------------------------------------------------------------------------
// pass 1: per-block partial (sum, sum of squares about a shift) in double -> partial[2*blocks]
__global__ void gln_partial_kernel(const float* __restrict__ x, long n, double* __restrict__ partial) {
    double s = 0.0, q = 0.0;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const double v = (double)x[i];
        s += v; q += v * v;
    }
    __shared__ double ss[32], qq[32];
    s = warp_sum_d(s); q = warp_sum_d(q);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { ss[w] = s; qq[w] = q; }
    __syncthreads();
    if (w == 0) {
        s = (l < (blockDim.x >> 5)) ? ss[l] : 0.0;
        q = (l < (blockDim.x >> 5)) ? qq[l] : 0.0;
        s = warp_sum_d(s); q = warp_sum_d(q);
        if (l == 0) { partial[2 * blockIdx.x] = s; partial[2 * blockIdx.x + 1] = q; }
    }
}
// pass 2 (one block): stats[0] = mean, stats[1] = 1/sqrt(var_unbiased + eps)
__global__ void gln_finalize_kernel(const double* __restrict__ partial, int nblocks, long n, float eps, float* __restrict__ stats) {
    double s = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < nblocks; i += blockDim.x) { s += partial[2 * i]; q += partial[2 * i + 1]; }
    __shared__ double ss[32], qq[32];
    s = warp_sum_d(s); q = warp_sum_d(q);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { ss[w] = s; qq[w] = q; }
    __syncthreads();
    if (threadIdx.x == 0) {
        s = 0.0; q = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { s += ss[i]; q += qq[i]; }
        const double mean = s / (double)n;
        const double var = (q - s * mean) / (double)(n > 1 ? n - 1 : 1);   // unbiased (torch.var default)
        stats[0] = (float)mean;
        stats[1] = (float)(1.0 / sqrt(var + (double)eps));
    }
}
__device__ __forceinline__ float silu_f(float v) { return v / (1.f + expf(-v)); }
__global__ void gln_apply_kernel(const float* __restrict__ x, const float* __restrict__ stats, float* __restrict__ y, long n, int silu) {
    const float mean = stats[0], rstd = stats[1];
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        float v = (x[i] - mean) * rstd;
        if (silu) v = silu_f(v);
        y[i] = v;
    }
}
// backward: xhat = (x-mean)*rstd ; y = silu?(xhat).  g = dy * silu'(xhat) (or dy).
//   dx = rstd * (g - mean(g) - xhat * sum(g*xhat)/(n-1))
__global__ void gln_bwd_partial_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ stats,
                                       long n, int silu, double* __restrict__ partial) {
    const float mean = stats[0], rstd = stats[1];
    double s = 0.0, q = 0.0;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const float xh = (x[i] - mean) * rstd;
        float g = dy[i];
        if (silu) { const float sg = 1.f / (1.f + expf(-xh)); g *= sg * (1.f + xh * (1.f - sg)); }
        s += (double)g; q += (double)g * (double)xh;
    }
    __shared__ double ss[32], qq[32];
    s = warp_sum_d(s); q = warp_sum_d(q);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { ss[w] = s; qq[w] = q; }
    __syncthreads();
    if (w == 0) {
        s = (l < (blockDim.x >> 5)) ? ss[l] : 0.0;
        q = (l < (blockDim.x >> 5)) ? qq[l] : 0.0;
        s = warp_sum_d(s); q = warp_sum_d(q);
        if (l == 0) { partial[2 * blockIdx.x] = s; partial[2 * blockIdx.x + 1] = q; }
    }
}
__global__ void gln_bwd_reduce_kernel(const double* __restrict__ partial, int nblocks, double* __restrict__ sums) {
    double s = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < nblocks; i += blockDim.x) { s += partial[2 * i]; q += partial[2 * i + 1]; }
    __shared__ double ss[32], qq[32];
    s = warp_sum_d(s); q = warp_sum_d(q);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) { ss[w] = s; qq[w] = q; }
    __syncthreads();
    if (threadIdx.x == 0) {
        s = 0.0; q = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { s += ss[i]; q += qq[i]; }
        sums[0] = s; sums[1] = q;
    }
}
__global__ void gln_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ stats,
                                     const double* __restrict__ sums, float* __restrict__ dx, long n, int silu) {
    const float mean = stats[0], rstd = stats[1];
    const float gmean = (float)(sums[0] / (double)n);
    const float gx = (float)(sums[1] / (double)(n > 1 ? n - 1 : 1));
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const float xh = (x[i] - mean) * rstd;
        float g = dy[i];
        if (silu) { const float sg = 1.f / (1.f + expf(-xh)); g *= sg * (1.f + xh * (1.f - sg)); }
        dx[i] = rstd * (g - gmean - xh * gx);
    }
}

// ---------------------------------------------------------------------------------------------------
// per-row LayerNorm with affine (nn.LayerNorm / openfold LayerNorm), one warp per row
// ---------------------------------------------------------------------------------------------------
// Column sums over all rows in one fixed order (no atomics, so the result is the same from run to run): one CTA per 32
// columns, 32 row lanes; lane r adds rows r, r + 32, ... in turn, then the 32 lane sums are added in lane order.
__global__ void __launch_bounds__(1024) colsum_kernel(const float* __restrict__ x, long R, long C, long ld, int pre_relu,
                                                      const float* __restrict__ gate, const float* __restrict__ gate_sub, long ldg,
                                                      float* __restrict__ colsum) {
    __shared__ float red[32][33];
    const int tx = threadIdx.x, ty = threadIdx.y;
    const long c = (long)blockIdx.x * 32 + tx;
    float s = 0.f;
    if (c < C) {
        for (long r = ty; r < R; r += 32) {
            float v = x[r * ld + c];
            if (pre_relu) v = fmaxf(v, 0.f);
            if (gate) v = gate_open(gate, gate_sub, r * ldg + c) ? v : 0.f;
            s += v;
        }
    }
    red[ty][tx] = s;
    __syncthreads();
    if (ty == 0 && c < C) {
        float t = 0.f;
        for (int i = 0; i < 32; ++i) t += red[i][tx];
        colsum[c] += t;
    }
}

// LayerNorm weight / bias gradients dw[c] += sum_r dy[r][c] xhat[r][c], db[c] += sum_r dy[r][c], in the fixed order of
// colsum_kernel.
__global__ void __launch_bounds__(1024) row_ln_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                            const float* __restrict__ stats, float* __restrict__ dw,
                                                            float* __restrict__ db, long rows, int C) {
    __shared__ float red_w[32][33], red_b[32][33];
    const int tx = threadIdx.x, ty = threadIdx.y;
    const long c = (long)blockIdx.x * 32 + tx;
    float sw = 0.f, sb = 0.f;
    if (c < C) {
        for (long r = ty; r < rows; r += 32) {
            const float g = dy[r * C + c];
            const float xh = (x[r * C + c] - stats[2 * r]) * stats[2 * r + 1];
            sw += g * xh;
            sb += g;
        }
    }
    red_w[ty][tx] = sw;
    red_b[ty][tx] = sb;
    __syncthreads();
    if (ty == 0 && c < C) {
        float tw = 0.f, tb = 0.f;
        for (int i = 0; i < 32; ++i) { tw += red_w[i][tx]; tb += red_b[i][tx]; }
        dw[c] += tw;
        db[c] += tb;
    }
}

__global__ void row_ln_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                  float* __restrict__ y, float* __restrict__ stats, long rows, int C, float eps) {
    const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const float* xr = x + row * C;
    float s = 0.f;
    for (int c = lane; c < C; c += 32) s += xr[c];
    const float mean = warp_sum(s) / C;
    float q = 0.f;
    for (int c = lane; c < C; c += 32) { const float d = xr[c] - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) / C + eps);
    for (int c = lane; c < C; c += 32) y[row * C + c] = (xr[c] - mean) * rstd * w[c] + b[c];
    if (lane == 0) { stats[2 * row] = mean; stats[2 * row + 1] = rstd; }
}
__global__ void row_ln_bwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ dy,
                                  const float* __restrict__ stats, float* __restrict__ dx, float* __restrict__ dw,
                                  float* __restrict__ db, long rows, int C) {
    const long row = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    const float mean = stats[2 * row], rstd = stats[2 * row + 1];
    const float* xr = x + row * C;
    const float* gr = dy + row * C;
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < C; c += 32) {
        const float xh = (xr[c] - mean) * rstd, g = gr[c] * w[c];
        s1 += g; s2 += g * xh;
    }
    s1 = warp_sum(s1) / C; s2 = warp_sum(s2) / C;
    for (int c = lane; c < C; c += 32) {
        const float xh = (xr[c] - mean) * rstd, g = gr[c] * w[c];
        dx[row * C + c] = rstd * (g - s1 - xh * s2);
    }
}

}  // namespace
}  // namespace dfold

using namespace dfold;

extern "C" const char* dfold_last_error(void) { return g_err; }
extern "C" int dfold_abi_version(void) { return 4; }

// id of the CUDA-graph capture `stream` is recording into (0 when the stream is not capturing).  The host side keys
// its cached operand planes on it: planes built inside one capture must never be reused by another graph.
extern "C" int dfold_capture_id(void* stream, unsigned long long* id_out) {
    DFOLD_REQUIRE(id_out != nullptr, "dfold_capture_id: null output");
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    unsigned long long id = 0;
    cudaError_t e = cudaStreamGetCaptureInfo(as_stream(stream), &st, &id);
    DFOLD_REQUIRE(e == cudaSuccess, "dfold_capture_id: %s", cudaGetErrorString(e));
    *id_out = (st == cudaStreamCaptureStatusActive) ? id : 0ull;
    return 0;
}

namespace {
int split2d(const float* x, long R, long C, long ld, int pre_relu, const float* gate, const float* gate_sub, long ldg,
            uint16_t* hi, uint16_t* lo, long ldo, long cpad, uint16_t* hi_t, uint16_t* lo_t, long ldt, long rpad,
            float* colsum, void* stream) {
    DFOLD_REQUIRE(R > 0 && C > 0, "dfold_split2d: empty input");
    DFOLD_REQUIRE((hi == nullptr) == (lo == nullptr) && (hi_t == nullptr) == (lo_t == nullptr), "dfold_split2d: hi/lo must come in pairs");
    DFOLD_REQUIRE(hi == nullptr || (cpad >= C && ldo >= cpad), "dfold_split2d: need C <= cpad <= ldo");
    DFOLD_REQUIRE(hi_t == nullptr || (rpad >= R && ldt >= rpad), "dfold_split2d: need R <= rpad <= ldt");
    // the grid covers the padded extents so the padding columns/rows are written as zeros
    const long cols = (hi && cpad > C) ? cpad : C;
    const long rows = (hi_t && rpad > R) ? rpad : R;
    if (colsum) {
        colsum_kernel<<<(unsigned)cdiv(C, 32), dim3(32, 32), 0, as_stream(stream)>>>(x, R, C, ld, pre_relu, gate, gate_sub, ldg, colsum);
        if (check_launch("colsum_kernel")) return 1;
    }
    if (!hi && !hi_t) return 0;         // column sums only (a bias gradient without operand planes)
    if (hi && !hi_t && (ld & 3) == 0 && (ldo & 3) == 0 && (cpad & 3) == 0 && (!gate || (ldg & 3) == 0) &&
        ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(gate) | reinterpret_cast<uintptr_t>(gate_sub)) & 15) == 0 &&
        ((reinterpret_cast<uintptr_t>(hi) | reinterpret_cast<uintptr_t>(lo)) & 7) == 0) {
        const long c4n = cpad / 4, n = R * c4n;
        split2d_vec_kernel<<<(unsigned)cdiv(n, 256), 256, 0, as_stream(stream)>>>(x, R, C, ld, pre_relu, gate, gate_sub, ldg, hi, lo,
                                                                                   ldo, c4n);
        return check_launch("split2d_vec_kernel");
    }
    dim3 grid((unsigned)cdiv(cols, 32), (unsigned)cdiv(rows, 32));
    split2d_kernel<<<grid, dim3(32, 8), 0, as_stream(stream)>>>(x, R, C, ld, pre_relu, gate, gate_sub, ldg, hi, lo, ldo, cpad,
                                                                hi_t, lo_t, ldt, rpad);
    return check_launch("split2d_kernel");
}
}  // namespace

// hi/lo: [R][ldo], columns [C, cpad) zero-filled.  hi_t/lo_t: [C][ldt], columns [R, rpad) zero-filled.
extern "C" int dfold_split2d(const float* x, long R, long C, long ld, int pre_relu, const float* gate, long ldg,
                             uint16_t* hi, uint16_t* lo, long ldo, long cpad, uint16_t* hi_t, uint16_t* lo_t, long ldt, long rpad,
                             float* colsum, void* stream) {
    return split2d(x, R, C, ld, pre_relu, gate, nullptr, ldg, hi, lo, ldo, cpad, hi_t, lo_t, ldt, rpad, colsum, stream);
}

// dfold_split2d with the gate of a residual layer: an element passes where (out - residual) > 0 (both [R][ldg]).
extern "C" int dfold_split2d_residual_gate(const float* x, long R, long C, long ld, int pre_relu, const float* out,
                                           const float* residual, long ldg, uint16_t* hi, uint16_t* lo, long ldo, long cpad,
                                           uint16_t* hi_t, uint16_t* lo_t, long ldt, long rpad, float* colsum, void* stream) {
    DFOLD_REQUIRE(out != nullptr && residual != nullptr, "dfold_split2d_residual_gate: out and residual are required");
    return split2d(x, R, C, ld, pre_relu, out, residual, ldg, hi, lo, ldo, cpad, hi_t, lo_t, ldt, rpad, colsum, stream);
}

extern "C" int dfold_conv_weight_prep(const float* w, int O, int I, int T, uint16_t* f_hi, uint16_t* f_lo, long ldi,
                                      uint16_t* d_hi, uint16_t* d_lo, long ldo, void* stream) {
    // the CTA stages a 32 x 32 x T tile in 32 * (32 T + 1) * 4 B of shared memory: T = 56 takes 229,504 B, T = 57 would take
    // 233,600 B, more than the 227 KB (232,448 B) a Hopper block can reserve
    DFOLD_REQUIRE(O > 0 && I > 0 && T > 0 && T <= 56, "dfold_conv_weight_prep: bad shape (need O, I > 0 and 1 <= T <= 56)");
    DFOLD_REQUIRE(ldi >= I && (d_hi == nullptr || ldo >= O), "dfold_conv_weight_prep: bad leading dims");
    dim3 grid((unsigned)cdiv(I, 32), (unsigned)cdiv(O, 32));
    const size_t smem = (size_t)32 * (32 * T + 1) * sizeof(uint32_t);
    static SmemCfg cfg;
    if (ensure_dyn_smem(conv_weight_prep_kernel, smem, cfg, "conv_weight_prep_kernel")) return 1;
    conv_weight_prep_kernel<<<grid, 256, smem, as_stream(stream)>>>(w, O, I, T, f_hi, f_lo, ldi, d_hi, d_lo, ldo);
    return check_launch("conv_weight_prep_kernel");
}

extern "C" int dfold_taps_to_param(const float* g, int O, int I, int T, float* out, int accumulate, void* stream) {
    DFOLD_REQUIRE(O > 0 && I > 0 && T > 0 && T <= 64, "dfold_taps_to_param: bad shape");
    dim3 grid((unsigned)cdiv(I, 64), (unsigned)O);
    taps_to_param_kernel<<<grid, 256, T * 65 * sizeof(float), as_stream(stream)>>>(g, O, I, T, out, accumulate);
    return check_launch("taps_to_param_kernel");
}

// Strides are in elements: *_rs row, *_cs column, *_bs / *_bs2 outer / inner batch.  C = act(alpha*A.B^T + bias) + beta*R.
// ksplit > 1 splits the K range over extra CTAs and atomically accumulates into a zeroed C (the summation order, and with
// it the last bits, then varies from run to run; the package's own callers split K with batched partials instead).
extern "C" int dfold_sgemm(const float* A, long a_rs, long a_cs, long a_bs, long a_bs2,
                           const float* B, long b_rs, long b_cs, long b_bs, long b_bs2,
                           float* C, long c_rs, long c_cs, long c_bs, long c_bs2,
                           const float* R, long r_rs, long r_cs, long r_bs, long r_bs2,
                           const float* bias, int batch, int batch2, int M, int N, int K, float alpha, float beta, int act,
                           int pre_relu, int ksplit, void* stream) {
    DFOLD_REQUIRE(batch > 0 && batch2 > 0 && M > 0 && N > 0 && K >= 0 && ksplit >= 1, "dfold_sgemm: empty problem");
    DFOLD_REQUIRE((long)batch * batch2 * ksplit <= 65535, "dfold_sgemm: batch too large (%d x %d x %d)", batch, batch2, ksplit);
    DFOLD_REQUIRE(ksplit == 1 || (bias == nullptr && R == nullptr && act == 0), "dfold_sgemm: split-K takes no epilogue (C must be zeroed)");
    SgemmParams p{A, a_rs, a_cs, a_bs, a_bs2, B, b_rs, b_cs, b_bs, b_bs2, C, c_rs, c_cs, c_bs, c_bs2,
                  R, r_rs, r_cs, r_bs, r_bs2, bias, batch2, ksplit, M, N, K, alpha, beta, act, pre_relu};
    dim3 grid((unsigned)cdiv(N, 64), (unsigned)cdiv(M, 64), (unsigned)(batch * batch2 * ksplit));
    sgemm_kernel<<<grid, 256, 0, as_stream(stream)>>>(p);
    return check_launch("sgemm_kernel");
}

// workspace: at least 2*1024 + 2 doubles
extern "C" int dfold_global_layernorm_fwd(const float* x, float* y, float* stats, double* workspace, long n, float eps, int silu, void* stream) {
    DFOLD_REQUIRE(n > 1, "dfold_global_layernorm_fwd: need at least 2 elements");
    const int blocks = (int)(cdiv(n, 256 * 8) < 1024 ? cdiv(n, 256 * 8) : 1024);
    cudaStream_t st = as_stream(stream);
    gln_partial_kernel<<<blocks, 256, 0, st>>>(x, n, workspace);
    gln_finalize_kernel<<<1, 256, 0, st>>>(workspace, blocks, n, eps, stats);
    gln_apply_kernel<<<(int)(cdiv(n, 256 * 4) < 4096 ? cdiv(n, 256 * 4) : 4096), 256, 0, st>>>(x, stats, y, n, silu);
    return check_launch("global_layernorm_fwd");
}

extern "C" int dfold_global_layernorm_bwd(const float* x, const float* dy, const float* stats, double* workspace, float* dx, long n, int silu, void* stream) {
    DFOLD_REQUIRE(n > 1, "dfold_global_layernorm_bwd: need at least 2 elements");
    const int blocks = (int)(cdiv(n, 256 * 8) < 1024 ? cdiv(n, 256 * 8) : 1024);
    cudaStream_t st = as_stream(stream);
    gln_bwd_partial_kernel<<<blocks, 256, 0, st>>>(x, dy, stats, n, silu, workspace);
    gln_bwd_reduce_kernel<<<1, 256, 0, st>>>(workspace, blocks, workspace + 2048);
    gln_bwd_apply_kernel<<<(int)(cdiv(n, 256 * 4) < 4096 ? cdiv(n, 256 * 4) : 4096), 256, 0, st>>>(x, dy, stats, workspace + 2048, dx, n, silu);
    return check_launch("global_layernorm_bwd");
}

extern "C" int dfold_row_layernorm_fwd(const float* x, const float* w, const float* b, float* y, float* stats, long rows, int C, float eps, void* stream) {
    DFOLD_REQUIRE(rows > 0 && C > 0, "dfold_row_layernorm_fwd: empty input");
    row_ln_fwd_kernel<<<(unsigned)cdiv(rows, 8), 256, 0, as_stream(stream)>>>(x, w, b, y, stats, rows, C, eps);
    return check_launch("row_ln_fwd_kernel");
}

extern "C" int dfold_row_layernorm_bwd(const float* x, const float* w, const float* dy, const float* stats, float* dx, float* dw, float* db,
                                       long rows, int C, void* stream) {
    DFOLD_REQUIRE(rows > 0 && C > 0, "dfold_row_layernorm_bwd: empty input");
    row_ln_bwd_kernel<<<(unsigned)cdiv(rows, 8), 256, 0, as_stream(stream)>>>(x, w, dy, stats, dx, dw, db, rows, C);
    if (check_launch("row_ln_bwd_kernel")) return 1;
    row_ln_wgrad_kernel<<<(unsigned)cdiv(C, 32), dim3(32, 32), 0, as_stream(stream)>>>(x, dy, stats, dw, db, rows, C);
    return check_launch("row_ln_wgrad_kernel");
}

// ---------------------------------------------------------------------------------------------------
// Adam (amsgrad) over flat fp32 buffers: the optimizer of the reference trainer (torch.optim.Adam(amsgrad=True),
// train_DFOLD_dynamics.py:412) for the graph-captured step of dynamicpdb_b200/train_step.py.  One pass over
// {param, grad, exp_avg, exp_avg_sq, max_exp_avg_sq}: 36 bytes per element instead of the ~90 of the multi-tensor kernels.
// `step` lives on the device (float; incremented by adam_tick_kernel) so the update is CUDA-graph capturable.
// ---------------------------------------------------------------------------------------------------
namespace dfold {
namespace {
__global__ void adam_tick_kernel(float* step) { *step += 1.f; }

// kClip: the gradient is ((g * gscale) * *coef), the order of DDP's mean followed by clip_grad_norm_'s mul_(coef).
// kDevLr: the learning rate is read from device memory (*dlr, written by lr_schedule_kernel) instead of the argument lr.
template <bool kClip, bool kDevLr>
__global__ void __launch_bounds__(256) adam_amsgrad_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                           float* __restrict__ v, float* __restrict__ vmax, long n4,
                                                           const float* __restrict__ step, float lr, float b1, float b2, float eps,
                                                           float gscale, const float* __restrict__ coef,
                                                           const float* __restrict__ dlr) {
    const float t = *step;
    const float bc1 = 1.f - powf(b1, t), bc2 = 1.f - powf(b2, t);
    const float step_size = (kDevLr ? *dlr : lr) / bc1, inv_bc2_sqrt = 1.f / sqrtf(bc2);
    const float c = kClip ? *coef : 1.f;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
        float4 P = reinterpret_cast<float4*>(p)[i];
        float4 G = reinterpret_cast<const float4*>(g)[i];
        G.x *= gscale; G.y *= gscale; G.z *= gscale; G.w *= gscale;      // 1 / world_size of the data-parallel mean
        if (kClip) { G.x *= c; G.y *= c; G.z *= c; G.w *= c; }
        float4 M = reinterpret_cast<float4*>(m)[i], V = reinterpret_cast<float4*>(v)[i], X = reinterpret_cast<float4*>(vmax)[i];
        float* pp = &P.x; const float* gg = &G.x; float* mm = &M.x; float* vv = &V.x; float* xx = &X.x;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            mm[c] = mm[c] + (gg[c] - mm[c]) * (1.f - b1);                  // exp_avg.lerp_(grad, 1 - beta1)
            vv[c] = vv[c] * b2 + (1.f - b2) * gg[c] * gg[c];
            xx[c] = fmaxf(xx[c], vv[c]);
            pp[c] = pp[c] - step_size * mm[c] / (sqrtf(xx[c]) * inv_bc2_sqrt + eps);
        }
        reinterpret_cast<float4*>(p)[i] = P;
        reinterpret_cast<float4*>(m)[i] = M;
        reinterpret_cast<float4*>(v)[i] = V;
        reinterpret_cast<float4*>(vmax)[i] = X;
    }
}

// ---------------------------------------------------------------------------------------------------
// Global L2 norm of the flat gradient and the clipping coefficient of torch.nn.utils.clip_grad_norm_ (norm_type 2), the
// optimizer-side option of the reference trainer (train_DFOLD_dynamics.py:665).  The order of the sum depends on n only, not
// on the device, so every run and every data-parallel rank (all reduce the same all-reduced buffer) gets the same bits:
// CTA b of grad_norm_blocks(n / 4) has thread t add, in turn, the squares of float4s b 256 + t, + 256 blocks, ... in fp64
// (the square of an fp32 value is exact there); then the 32 lanes by xor butterfly and the 8 warp sums in warp order.
// ---------------------------------------------------------------------------------------------------
constexpr int kNormThreads = 256, kNormMaxBlocks = 1024;

static inline int grad_norm_blocks(long n4) {
    return (int)(cdiv(n4, kNormThreads) < kNormMaxBlocks ? cdiv(n4, kNormThreads) : kNormMaxBlocks);
}

// sum over the CTA's 256 threads (valid in thread 0)
__device__ __forceinline__ double norm_block_sum(double s) {
    __shared__ double red[kNormThreads / 32];
    s = warp_sum_d(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kNormThreads / 32; ++w) t += red[w];
    return t;
}

__global__ void __launch_bounds__(kNormThreads) grad_sqnorm_partial_kernel(const float* __restrict__ g, long n4,
                                                                           double* __restrict__ partial) {
    double s = 0.0;
    for (long i = (long)blockIdx.x * kNormThreads + threadIdx.x; i < n4; i += (long)gridDim.x * kNormThreads) {
        const float4 G = reinterpret_cast<const float4*>(g)[i];
        const double x = G.x, y = G.y, z = G.z, w = G.w;
        s = fma(x, x, s); s = fma(y, y, s); s = fma(z, z, s); s = fma(w, w, s);
    }
    s = norm_block_sum(s);
    if (threadIdx.x == 0) partial[blockIdx.x] = s;
}

// One CTA: thread t adds partials t, t + 256, ... in turn, then as above.  total = fp32(sqrt(sum) gscale), and the
// coefficient in fp32 as torch evaluates max_norm / (total + 1e-6) (Tensor.__rtruediv__: reciprocal, then the product)
// clamped to at most 1, where a NaN stays NaN as in torch.clamp.
__global__ void __launch_bounds__(kNormThreads) grad_norm_finalize_kernel(const double* __restrict__ partial, int nblocks,
                                                                          float gscale, float max_norm,
                                                                          float* __restrict__ total, float* __restrict__ coef) {
    double s = 0.0;
    for (int i = threadIdx.x; i < nblocks; i += kNormThreads) s += partial[i];
    s = norm_block_sum(s);
    if (threadIdx.x == 0) {
        const float tn = (float)(sqrt(s) * (double)gscale);
        const float c = __fmul_rn(__frcp_rn(__fadd_rn(tn, 1e-6f)), max_norm);
        *total = tn;
        *coef = (c > 1.f) ? 1.f : c;
    }
}

// ---------------------------------------------------------------------------------------------------
// The AlphaFold learning-rate schedule (openfold/utils/lr_schedulers.py AlphaFoldLRScheduler.get_lr, the scheduler the
// reference trainer imports, train_DFOLD_dynamics.py:56,652) at last_epoch = *step, the optimizer steps taken so far.  One
// thread, evaluated in fp64 in Python's order with every operation rounded on its own (no contraction), then rounded to fp32
// once: the value a Python float lr becomes when it is passed to the fp32 Adam.  The decay power decay ** e (integer e >= 1)
// goes through pow as Python's float.__pow__ does.
// ---------------------------------------------------------------------------------------------------
__global__ void lr_schedule_kernel(const float* __restrict__ step, double base_lr, double max_lr, long warmup, long start,
                                   long every, double decay, float* __restrict__ lr) {
    const long s = (long)*step;
    double v;
    if (s <= warmup)
        v = __dadd_rn(base_lr, __dmul_rn(__ddiv_rn((double)s, (double)warmup), max_lr));
    else if (s > start)
        v = __dmul_rn(max_lr, pow(decay, (double)((s - start) / every + 1)));
    else
        v = max_lr;
    *lr = (float)v;
}
}  // namespace

static int adam_launch(bool clip, float* param, const float* grad, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq,
                       long n, float* step, int tick, float lr, float beta1, float beta2, float eps, float grad_scale,
                       const float* coef, const float* dlr, cudaStream_t st) {
    if (tick) adam_tick_kernel<<<1, 1, 0, st>>>(step);            // chunked callers advance the step once per optimizer step
    const long n4 = n / 4;
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
        sms = 132;
    const long cap = 16L * sms;                                     // 16 CTAs of 256 threads per SM, grid-stride beyond
    const int blocks = (int)(cdiv(n4, 256) < cap ? cdiv(n4, 256) : cap);
#define DFOLD_ADAM(CLIP, DLR)                                                                                                  \
    adam_amsgrad_kernel<CLIP, DLR><<<blocks, 256, 0, st>>>(param, grad, exp_avg, exp_avg_sq, max_exp_avg_sq, n4, step, lr, beta1, \
                                                           beta2, eps, grad_scale, coef, dlr)
    if (dlr != nullptr) {
        if (clip) DFOLD_ADAM(true, true); else DFOLD_ADAM(false, true);
    } else {
        if (clip) DFOLD_ADAM(true, false); else DFOLD_ADAM(false, false);
    }
#undef DFOLD_ADAM
    return check_launch("adam_amsgrad_kernel");
}
}  // namespace dfold

// n must be a multiple of 4 and the buffers 16-byte aligned (train_step.py pads its flat buffers).
extern "C" int dfold_adam_amsgrad(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq, long n,
                                  float* step, int tick, float lr, float beta1, float beta2, float eps, float grad_scale, void* stream) {
    DFOLD_REQUIRE(n > 0 && n % 4 == 0, "dfold_adam_amsgrad: n must be a positive multiple of 4");
    return dfold::adam_launch(false, param, grad, exp_avg, exp_avg_sq, max_exp_avg_sq, n, step, tick, lr, beta1, beta2, eps,
                              grad_scale, nullptr, nullptr, dfold::as_stream(stream));
}

extern "C" int dfold_adam_amsgrad_clip(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq,
                                       long n, float* step, int tick, float lr, float beta1, float beta2, float eps, float grad_scale,
                                       const float* coef, void* stream) {
    DFOLD_REQUIRE(n > 0 && n % 4 == 0, "dfold_adam_amsgrad_clip: n must be a positive multiple of 4");
    DFOLD_REQUIRE(coef != nullptr, "dfold_adam_amsgrad_clip: null coefficient");
    return dfold::adam_launch(true, param, grad, exp_avg, exp_avg_sq, max_exp_avg_sq, n, step, tick, lr, beta1, beta2, eps,
                              grad_scale, coef, nullptr, dfold::as_stream(stream));
}

// lr: DEVICE fp32 scalar; coef: nullable (no clipping).
extern "C" int dfold_adam_amsgrad_dlr(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq,
                                      long n, float* step, int tick, const float* lr, float beta1, float beta2, float eps,
                                      float grad_scale, const float* coef, void* stream) {
    DFOLD_REQUIRE(n > 0 && n % 4 == 0, "dfold_adam_amsgrad_dlr: n must be a positive multiple of 4");
    DFOLD_REQUIRE(lr != nullptr, "dfold_adam_amsgrad_dlr: null learning rate");
    return dfold::adam_launch(coef != nullptr, param, grad, exp_avg, exp_avg_sq, max_exp_avg_sq, n, step, tick, 0.f, beta1, beta2,
                              eps, grad_scale, coef, lr, dfold::as_stream(stream));
}

extern "C" int dfold_lr_schedule(const float* step, double base_lr, double max_lr, long warmup_no_steps,
                                 long start_decay_after_n_steps, long decay_every_n_steps, double decay_factor, float* lr,
                                 void* stream) {
    DFOLD_REQUIRE(step != nullptr && lr != nullptr, "dfold_lr_schedule: null step or lr");
    DFOLD_REQUIRE(warmup_no_steps > 0 && decay_every_n_steps > 0 && warmup_no_steps <= start_decay_after_n_steps,
                  "dfold_lr_schedule: needs 0 < warmup_no_steps <= start_decay_after_n_steps and decay_every_n_steps > 0");
    DFOLD_REQUIRE(max_lr > 0.0 && max_lr < INFINITY, "dfold_lr_schedule: max_lr must be positive and finite");
    dfold::lr_schedule_kernel<<<1, 1, 0, dfold::as_stream(stream)>>>(step, base_lr, max_lr, warmup_no_steps,
                                                                     start_decay_after_n_steps, decay_every_n_steps, decay_factor, lr);
    return dfold::check_launch("lr_schedule_kernel");
}

// partial: workspace of at least 1024 doubles.
extern "C" int dfold_grad_norm(const float* grad, long n, float grad_scale, float max_norm, double* partial, float* total,
                               float* coef, void* stream) {
    DFOLD_REQUIRE(n > 0 && n % 4 == 0, "dfold_grad_norm: n must be a positive multiple of 4");
    DFOLD_REQUIRE(max_norm > 0.f, "dfold_grad_norm: max_norm must be positive (inf reports the norm without clipping)");
    DFOLD_REQUIRE(partial != nullptr && total != nullptr && coef != nullptr, "dfold_grad_norm: null workspace or output");
    cudaStream_t st = dfold::as_stream(stream);
    const long n4 = n / 4;
    const int blocks = dfold::grad_norm_blocks(n4);
    dfold::grad_sqnorm_partial_kernel<<<blocks, dfold::kNormThreads, 0, st>>>(grad, n4, partial);
    if (dfold::check_launch("grad_sqnorm_partial_kernel")) return 1;
    dfold::grad_norm_finalize_kernel<<<1, dfold::kNormThreads, 0, st>>>(partial, blocks, grad_scale, max_norm, total, coef);
    return dfold::check_launch("grad_norm_finalize_kernel");
}
