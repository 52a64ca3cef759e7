// Auxiliary structure losses of the DFOLDv2 score network (reference train_DFOLD_dynamics.py:1316-1364), value and
// gradient, without an O((5N)^2) buffer.
//
// Over the 5 backbone atoms (N, CA, C, CB, O) of every residue of EVERY frame f (A = 5N atoms per frame):
//   bb_atom_loss[f]  = sum_i |pred_i - gt_i|^2 bm_i / (sum_i bm_i + 1e-10) * w_bb * (t < t_bb) * w_aux,
//                      bm_i = any(gt_i != 0) * lm(i)                                                   (:1327-1335)
//   dist_mat_loss[f] = sum_ij (g_ij - p_ij)^2 m_ij / (sum_ij m_ij - N) * w_dm * (t < t_dm) * w_aux,       (:1344-1364)
//                      g_ij = |gt_i - gt_j| lm(i), p_ij = |pred_i - pred_j| lm(i), m_ij = lm(i) rm(j) (g_ij < 6)
// with lm = res_mask * (1 - fixed_mask) and rm = res_mask of the atom's residue.  m is not symmetric, but both distances
// are, so row i's gradient collects the (i, j) and (j, i) terms: d/d pred_i = sum_j -2 u_ij [(g_ij - p_ij) lm(i) m_ij +
// (g_ji - p_ji) lm(j) m_ji], u_ij = (pred_i - pred_j) / |pred_i - pred_j|.  Each CTA owns AT rows of one frame and
// streams every column tile through shared memory, so every row finishes its own gradient without atomics.  A vector
// norm has gradient 0 at 0 (torch's convention), so diagonal pairs and coincident atoms contribute 0.
//
// Kernel 1 writes each row's raw gradients and each CTA's fixed-order fp64 partial sums; kernel 2 reduces them per
// frame in a fixed order, applies the weights, the `t < filter` gates (read on the device) and the normalisation over
// non-empty frames (:1374-1375), and scales the gradient rows.  Results are bit-identical from run to run.
#include "common.cuh"

namespace dfold {
namespace {

constexpr int AT = 128;     // atoms per row tile (one per thread) and per staged column tile
constexpr int FT = 256;     // threads of the finishing kernel
constexpr int NP = 5;       // partials per (frame, row tile): dist num, dist mask, bb num, bb mask, frame non-empty
constexpr int MAX_NF = 2048;

struct AuxParams {
    const float* pred;      // [nf,N,37,3] predicted atom37 (atoms 0..4 read)
    const float* gt;        // [nf,N,37,3] ground-truth backbone (atoms 0..4 read)
    const double* res_mask; const double* fixed_mask;   // [nf,N]
    const double* t; int t_stride;                       // t[f * t_stride]
    int nf, N, tiles;
    double w_bb, t_bb, w_dm, t_dm, w_aux;
    double* part;           // [nf, tiles, NP]
    double* out;            // [2 + 2 nf]: bb, dist (normalised), bb[nf], dist[nf]
    double* d_bb; double* d_dm;                          // [nf,N,5,3]
};

__device__ double block_sum(double v, double* red) {
    v = warp_sum_d(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < AT / 32; ++w) s += red[w];
    return s;
}

__global__ void __launch_bounds__(AT) aux_rows_kernel(const AuxParams p) {
    __shared__ float sx[AT][3], sg[AT][3];
    __shared__ double slm[AT], srm[AT], red[AT / 32];
    const int f = blockIdx.y, N = p.N, A = 5 * N, tid = threadIdx.x;
    const int i = blockIdx.x * AT + tid;
    const float* P = p.pred + (long)f * N * 111;
    const float* G = p.gt + (long)f * N * 111;
    const double* rm = p.res_mask + (long)f * N;
    const double* fm = p.fixed_mask + (long)f * N;
    const bool row = i < A;
    double xi[3] = {0, 0, 0}, gi[3] = {0, 0, 0}, lmi = 0, rmi = 0;
    bool gnz = false;
    if (row) {
        const int r = i / 5, a = i % 5;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float g = G[(r * 37 + a) * 3 + c];
            xi[c] = P[(r * 37 + a) * 3 + c];
            gi[c] = g;
            gnz = gnz || (g != 0.0f);
        }
        rmi = rm[r];
        lmi = rmi * (1.0 - fm[r]);
    }
    double acc[3] = {0, 0, 0}, num = 0, cnt = 0;
    for (int j0 = 0; j0 < A; j0 += AT) {
        __syncthreads();
        const int j = j0 + tid;
        if (j < A) {
            const int r = j / 5, a = j % 5;
#pragma unroll
            for (int c = 0; c < 3; ++c) { sx[tid][c] = P[(r * 37 + a) * 3 + c]; sg[tid][c] = G[(r * 37 + a) * 3 + c]; }
            srm[tid] = rm[r];
            slm[tid] = rm[r] * (1.0 - fm[r]);
        }
        __syncthreads();
        if (!row) continue;
        const int nj = min(AT, A - j0);
        for (int jj = 0; jj < nj; ++jj) {
            const double lmj = slm[jj], wij = lmi * srm[jj], wji = lmj * rmi;
            if (wij == 0.0 && wji == 0.0) continue;
            const double g0 = gi[0] - sg[jj][0], g1 = gi[1] - sg[jj][1], g2 = gi[2] - sg[jj][2];
            const double gd2 = g0 * g0 + g1 * g1 + g2 * g2;
            // a counted direction with lm >= 1 is excluded once |gt_i - gt_j| >= 6: skip the square roots
            if (gd2 >= 36.01 && (wij == 0.0 || lmi >= 1.0) && (wji == 0.0 || lmj >= 1.0)) continue;
            const double gd = sqrt(gd2);
            const double mij = (gd * lmi < 6.0) ? wij : 0.0, mji = (gd * lmj < 6.0) ? wji : 0.0;
            if (mij == 0.0 && mji == 0.0) continue;
            const double d0 = xi[0] - sx[jj][0], d1 = xi[1] - sx[jj][1], d2 = xi[2] - sx[jj][2];
            const double pd = sqrt(d0 * d0 + d1 * d1 + d2 * d2);
            const double eij = gd * lmi - pd * lmi, eji = gd * lmj - pd * lmj;
            num += eij * eij * mij;
            cnt += mij;
            if (pd > 0.0) {
                const double k = -2.0 * (eij * lmi * mij + eji * lmj * mji) / pd;
                acc[0] += k * d0; acc[1] += k * d1; acc[2] += k * d2;
            }
        }
    }
    double bnum = 0, bcnt = 0;
    if (row) {
        const double bm = gnz ? lmi : 0.0;
        double* db = p.d_bb + ((long)f * A + i) * 3;
        double* dd = p.d_dm + ((long)f * A + i) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double e = xi[c] - gi[c];
            bnum += e * e * bm;
            db[c] = 2.0 * e * bm;
            dd[c] = acc[c];
        }
        bcnt = bm;
    }
    // frames with any unmasked residue (:1222 batch_loss_mask), counted once per frame by its first row tile
    bool any = false;
    if (blockIdx.x == 0)
        for (int r = tid; r < N; r += AT) any = any || (rm[r] != 0.0);
    const double nonempty = __syncthreads_or(any) ? 1.0 : 0.0;
    num = block_sum(num, red); cnt = block_sum(cnt, red); bnum = block_sum(bnum, red); bcnt = block_sum(bcnt, red);
    if (tid == 0) {
        double* q = p.part + ((long)f * p.tiles + blockIdx.x) * NP;
        q[0] = num; q[1] = cnt; q[2] = bnum; q[3] = bcnt; q[4] = blockIdx.x == 0 ? nonempty : 0.0;
    }
}

__global__ void __launch_bounds__(FT) aux_finish_kernel(const AuxParams p) {
    extern __shared__ double sv[];          // [nf] bb, [nf] dist, [nf] non-empty
    __shared__ double k_bb, k_dm;
    const int f = blockIdx.x, nf = p.nf, tid = threadIdx.x;
    // every CTA reduces every frame (a few thousand loads): the totals need all of them, and each CTA then scales its own
    // frame's rows without another launch
    for (int ff = tid; ff < nf; ff += FT) {
        double s[NP] = {0, 0, 0, 0, 0};
        for (int b = 0; b < p.tiles; ++b)
            for (int k = 0; k < NP; ++k) s[k] += p.part[((long)ff * p.tiles + b) * NP + k];
        const double t = p.t[(long)ff * p.t_stride];
        const double gbb = (t < p.t_bb) ? 1.0 : 0.0, gdm = (t < p.t_dm) ? 1.0 : 0.0;
        sv[ff] = s[2] / (s[3] + 1e-10) * p.w_bb * gbb * p.w_aux;
        sv[nf + ff] = s[0] / (s[1] - (double)p.N) * p.w_dm * gdm * p.w_aux;
        sv[2 * nf + ff] = s[4];
        if (ff == f) {
            k_bb = p.w_bb * gbb * p.w_aux / (s[3] + 1e-10);
            k_dm = p.w_dm * gdm * p.w_aux / (s[1] - (double)p.N);
        }
    }
    __syncthreads();
    double cnt = 0;
    for (int ff = 0; ff < nf; ++ff) cnt += sv[2 * nf + ff];
    // x.sum() / (batch_loss_mask.sum() + 1e-10): the count is an integer tensor, so torch forms the denominator in fp32
    const double inv = 1.0 / (double)((float)cnt + 1e-10f);
    if (f == 0 && tid == 0) {
        double bb = 0, dm = 0;
        for (int ff = 0; ff < nf; ++ff) {
            bb += sv[ff];
            dm += sv[nf + ff];
            p.out[2 + ff] = sv[ff];
            p.out[2 + nf + ff] = sv[nf + ff];
        }
        p.out[0] = bb * inv;
        p.out[1] = dm * inv;
    }
    const double sb = k_bb * inv, sd = k_dm * inv;
    const long n = 15L * p.N, base = (long)f * n;
    for (long e = tid; e < n; e += FT) {
        p.d_bb[base + e] *= sb;
        p.d_dm[base + e] *= sd;
    }
}

}  // namespace
}  // namespace dfold

using namespace dfold;

extern "C" int dfold_aux_loss_fwd(const float* pred_atom37, const float* gt_atom37, const double* res_mask,
                                  const double* fixed_mask, const double* t, int t_stride, int nf, int N, double w_bb,
                                  double t_bb, double w_dm, double t_dm, double w_aux, double* work, double* out,
                                  double* d_bb, double* d_dm, void* stream) {
    DFOLD_REQUIRE(nf > 0 && N > 0, "dfold_aux_loss_fwd: empty problem");
    DFOLD_REQUIRE(nf <= MAX_NF, "dfold_aux_loss_fwd: nf = %d > %d frames", nf, MAX_NF);
    DFOLD_REQUIRE(t_stride == 0 || t_stride == 1, "dfold_aux_loss_fwd: t_stride must be 0 or 1");
    AuxParams p;
    p.pred = pred_atom37; p.gt = gt_atom37; p.res_mask = res_mask; p.fixed_mask = fixed_mask; p.t = t;
    p.t_stride = t_stride; p.nf = nf; p.N = N; p.tiles = (int)cdiv(5L * N, AT);
    p.w_bb = w_bb; p.t_bb = t_bb; p.w_dm = w_dm; p.t_dm = t_dm; p.w_aux = w_aux;
    p.part = work; p.out = out; p.d_bb = d_bb; p.d_dm = d_dm;
    cudaStream_t s = as_stream(stream);
    aux_rows_kernel<<<dim3(p.tiles, nf), AT, 0, s>>>(p);
    int rc = check_launch("aux_rows_kernel");
    if (rc) return rc;
    aux_finish_kernel<<<nf, FT, 3 * nf * sizeof(double), s>>>(p);
    return check_launch("aux_finish_kernel");
}
