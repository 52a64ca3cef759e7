// Trajectory metrics of the evaluator on the device, all in fp64 (fp32 inputs are upcast, which is exact).
//
//   rigid_error_kernel   per-frame mean quaternion angle (degrees) and translation MAE of the predicted frames and of the
//                        "reference" baseline (ground-truth frame ref_frame, broadcast), one CTA per frame.  Replaces
//                        src/toolbox/rot_trans_error.py:7-73 as Experiment._calc_rot_trans_error calls it
//                        (train_DFOLD_dynamics.py:1549-1568).
//   atom_error_kernel    per-frame masked atom37 sums: MAE / MSE of eval_fn (:892-912) and rmsd_all / rmsd_ca of
//                        compute_validation_metrics_all (:99-146), one CTA per frame.
//   superimpose_kernel   batched Kabsch in fp64, one CTA per point set: SVDSuperimposer as eval_fn (:898-909) and
//                        openfold/utils/superimposition.py use it.
//   drmsd_tile_kernel +  dRMSD (openfold/utils/validation_metrics.py:17-36): one CTA per 64 x 64 tile of the pair grid of
//   drmsd_reduce_kernel  a point set writes one partial; one CTA reduces the partials and the mask counts.
//
// Every sum runs in a fixed order (per-thread strided loops, then a shared-memory tree of fixed shape; no atomics), so a
// second launch gives the same bits.  No value goes back to the host: every launch can be captured in a CUDA graph.
#include <math.h>

#include "common.cuh"

namespace dfold {
namespace {

constexpr int kThreads = 256;
constexpr int kTile = 64;
constexpr double kPi = 3.141592653589793;

__device__ __forceinline__ double ldv(const void* p, int f64, long k) {
    return f64 ? __ldg(static_cast<const double*>(p) + k) : (double)__ldg(static_cast<const float*>(p) + k);
}

// Sum of one double per thread over the CTA: a tree of fixed shape over red[kThreads] (every thread gets the result).
__device__ __forceinline__ double block_sum(double v, double* red) {
    red[threadIdx.x] = v;
    __syncthreads();
#pragma unroll
    for (int s = kThreads / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    const double r = red[0];
    __syncthreads();
    return r;
}

// A batch of point sets read in place: coordinate c of point i of set s is p[s * sstride + i * pstride + c];
// a mask entry is m[s * msstride + i * mpstride] (m == NULL: all ones).
struct PointSets {
    const void* a; int a64;
    const void* b; int b64;
    long sstride, pstride;
    const void* m; int m64;
    long msstride, mpstride;
};

__device__ __forceinline__ double ld_mask(const PointSets& P, long s, long i) {
    return P.m ? ldv(P.m, P.m64, s * P.msstride + i * P.mpstride) : 1.0;
}

// ------------------------------------------------------------------------------------------------------------
// Rigid errors.  rot_trans_error.py: q / |q| (normalize_quaternions :58-60), angle = degrees(2 acos(|clip(q1.q2, -1, 1)|))
// (:50-55), mean over residues (:63-73); translation MAE = mean |t1 - t2| over residues and xyz, NOT masked (:16).
// out [4][nf]: pred vs gt rotation, translation; gt[ref_frame] vs gt rotation, translation.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double quat_angle_deg(const double* a, const double* b) {
    const double na = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2] + a[3] * a[3]);
    const double nb = sqrt(b[0] * b[0] + b[1] * b[1] + b[2] * b[2] + b[3] * b[3]);
    double dot = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) dot += (a[k] / na) * (b[k] / nb);
    dot = fmin(fmax(dot, -1.0), 1.0);
    return 2.0 * acos(fabs(dot)) * (180.0 / kPi);
}

__global__ void __launch_bounds__(kThreads) rigid_error_kernel(const void* pred, int pred64, const void* gt, int gt64, int N,
                                                               int ref_frame, int nf, double* __restrict__ out) {
    __shared__ double red[kThreads];
    const int f = blockIdx.x;
    double rot = 0.0, tr = 0.0, rrot = 0.0, rtr = 0.0;
    for (int i = threadIdx.x; i < N; i += kThreads) {
        const long pi = ((long)f * N + i) * 7, ri = ((long)ref_frame * N + i) * 7;
        double qg[4], qp[4], qr[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            qg[k] = ldv(gt, gt64, pi + k);
            qp[k] = ldv(pred, pred64, pi + k);
            qr[k] = ldv(gt, gt64, ri + k);
        }
        rot += quat_angle_deg(qg, qp);
        rrot += quat_angle_deg(qg, qr);
#pragma unroll
        for (int c = 4; c < 7; ++c) {
            const double g = ldv(gt, gt64, pi + c);
            tr += fabs(g - ldv(pred, pred64, pi + c));
            rtr += fabs(g - ldv(gt, gt64, ri + c));
        }
    }
    rot = block_sum(rot, red);
    tr = block_sum(tr, red);
    rrot = block_sum(rrot, red);
    rtr = block_sum(rtr, red);
    if (threadIdx.x == 0) {
        out[f] = rot / (double)N;
        out[nf + f] = tr / (3.0 * N);
        out[2 * nf + f] = rrot / (double)N;
        out[3 * nf + f] = rtr / (3.0 * N);
    }
}

// ------------------------------------------------------------------------------------------------------------
// Atom errors over [nf][N][A][3] with mask [nf][N][A].  eval_fn (:892-912): the mask is expanded over xyz, so
// MAE = sum |gt - pred| m / (3 sum m), MSE = sum (gt - pred)^2 m / (3 sum m) (0 / 0 = NaN for an empty frame);
// drop_last_atom zeroes mask[nf-1][N-1][A-1] (eval_fn's `atom_mask[-1, -1, -1] = 0.0`).
// compute_validation_metrics_all (:113-146): rmsd_all = sqrt(sum (gt m - pred m)^2 / (sum m + 1e-4)), rmsd_ca the same
// over atom column 1 (CA).  out [6][nf]: mae, mse, rmsd_all, rmsd_ca, sum m, sum m over CA.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) atom_error_kernel(const void* pred, int pred64, const void* gt, int gt64,
                                                              const void* mask, int mask64, int N, int A, int drop_last_atom,
                                                              int nf, double* __restrict__ out) {
    __shared__ double red[kThreads];
    const int f = blockIdx.x;
    const long npts = (long)N * A, base = (long)f * npts;
    const long dropped = (drop_last_atom && f == nf - 1) ? npts - 1 : -1;
    double sabs = 0.0, ssq = 0.0, sall = 0.0, sca = 0.0, cnt = 0.0, cca = 0.0;
    for (long e = threadIdx.x; e < npts; e += kThreads) {
        const double m = e == dropped ? 0.0 : ldv(mask, mask64, base + e);
        const bool ca = e % A == 1;
        double q = 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double g = ldv(gt, gt64, 3 * (base + e) + c), p = ldv(pred, pred64, 3 * (base + e) + c);
            const double d = g - p;
            sabs += fabs(d) * m;
            ssq += d * d * m;
            const double dm = g * m - p * m;
            q += dm * dm;
        }
        sall += q;
        cnt += m;
        if (ca) { sca += q; cca += m; }
    }
    sabs = block_sum(sabs, red);
    ssq = block_sum(ssq, red);
    sall = block_sum(sall, red);
    sca = block_sum(sca, red);
    cnt = block_sum(cnt, red);
    cca = block_sum(cca, red);
    if (threadIdx.x == 0) {
        out[f] = sabs / (3.0 * cnt);
        out[nf + f] = ssq / (3.0 * cnt);
        out[2 * nf + f] = sqrt(sall / (cnt + 1e-4));
        out[3 * nf + f] = sqrt(sca / (cca + 1e-4));
        out[4 * nf + f] = cnt;
        out[5 * nf + f] = cca;
    }
}

// ------------------------------------------------------------------------------------------------------------
// Kabsch superposition of set b (coords) onto set a (reference): R, t minimising sum w |R b + t - a|^2.
// Method: Horn's quaternion key matrix.  With S = sum w (b - cb)(a - ca)^T (centred in a second pass: coordinates may
// sit 10^3 A from the origin, where the one-pass sum w b a^T - W cb ca^T cancels), the optimal unit quaternion is the
// eigenvector of the largest eigenvalue of the symmetric 4x4 matrix K(S).  A unit quaternion is always a proper rotation,
// so no determinant fix is needed, and a symmetric 4x4 eigenproblem is solved to full fp64 accuracy by a fixed number of
// cyclic Jacobi sweeps (no data-dependent iteration count, no 3x3 SVD sign bookkeeping).  Rank-deficient sets (1 or 2
// points, collinear or coplanar points) have a degenerate top eigenvalue; any unit vector of that eigenspace is an optimal
// rotation, and Jacobi returns one.  The RMSD is sqrt(sum w |R (b - cb) - (a - ca)|^2 / W), computed by applying R in a
// third pass (E0 - 2 lambda_max cancels for good fits).  W = 0: RMSD NaN, R = I, t = 0, coords = b.
// mask_mode: 0 no mask (w = 1), 1 w = mask (selection / weights), 2 coordinates multiplied by the mask, w = 1
// (compute_validation_metrics_all superimposes the zeroed masked CA positions too, train_DFOLD_dynamics.py:113-150).
// ------------------------------------------------------------------------------------------------------------
__device__ void jacobi4_top(double A[4][4], double q[4]) {
    double V[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) V[r][c] = r == c ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 12; ++sweep) {
#pragma unroll
        for (int p = 0; p < 3; ++p) {
#pragma unroll
            for (int r = p + 1; r < 4; ++r) {
                const double apq = A[p][r];
                if (apq == 0.0) continue;
                const double th = (A[r][r] - A[p][p]) / (2.0 * apq);
                const double t = fabs(th) < 1e150 ? (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0)) : 0.5 / th;
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const double akp = A[k][p], akq = A[k][r];
                    A[k][p] = c * akp - s * akq;
                    A[k][r] = s * akp + c * akq;
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const double apk = A[p][k], aqk = A[r][k];
                    A[p][k] = c * apk - s * aqk;
                    A[r][k] = s * apk + c * aqk;
                }
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const double vkp = V[k][p], vkq = V[k][r];
                    V[k][p] = c * vkp - s * vkq;
                    V[k][r] = s * vkp + c * vkq;
                }
            }
        }
    }
    int best = 0;
#pragma unroll
    for (int k = 1; k < 4; ++k)
        if (A[k][k] > A[best][best]) best = k;
    const double n = sqrt(V[0][best] * V[0][best] + V[1][best] * V[1][best] + V[2][best] * V[2][best] + V[3][best] * V[3][best]);
#pragma unroll
    for (int k = 0; k < 4; ++k) q[k] = V[k][best] / n;
}

struct SupOut { double* rmsd; double* rot; double* trans; double* coords; };

__global__ void __launch_bounds__(kThreads) superimpose_kernel(const PointSets P, int npts, int mask_mode, SupOut o) {
    __shared__ double red[kThreads];
    __shared__ double s_R[9];
    const long s = blockIdx.x;
    auto load = [&](long i, double* a, double* b, double& w) {
        const double m = mask_mode ? ld_mask(P, s, i) : 1.0;
        const long k = s * P.sstride + i * P.pstride;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            a[c] = ldv(P.a, P.a64, k + c);
            b[c] = ldv(P.b, P.b64, k + c);
            if (mask_mode == 2) { a[c] *= m; b[c] *= m; }
        }
        w = mask_mode == 1 ? m : 1.0;
    };
    // pass 1: weight and centroids
    double sw = 0.0, sa[3] = {0.0, 0.0, 0.0}, sb[3] = {0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < npts; i += kThreads) {
        double a[3], b[3], w;
        load(i, a, b, w);
        sw += w;
#pragma unroll
        for (int c = 0; c < 3; ++c) { sa[c] += w * a[c]; sb[c] += w * b[c]; }
    }
    const double W = block_sum(sw, red);
    double ca[3], cb[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) { ca[c] = block_sum(sa[c], red) / W; cb[c] = block_sum(sb[c], red) / W; }
    const bool empty = !(W != 0.0);
    // pass 2: centred covariance S[x][y] = sum w (b_x - cb_x)(a_y - ca_y)
    double S[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) S[k] = 0.0;
    if (!empty) {
        for (int i = threadIdx.x; i < npts; i += kThreads) {
            double a[3], b[3], w;
            load(i, a, b, w);
#pragma unroll
            for (int x = 0; x < 3; ++x)
#pragma unroll
                for (int y = 0; y < 3; ++y) S[3 * x + y] += w * (b[x] - cb[x]) * (a[y] - ca[y]);
        }
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) S[k] = block_sum(S[k], red);
    if (threadIdx.x == 0) {
        double q[4] = {1.0, 0.0, 0.0, 0.0};
        if (!empty) {
            const double xx = S[0], xy = S[1], xz = S[2], yx = S[3], yy = S[4], yz = S[5], zx = S[6], zy = S[7], zz = S[8];
            double K[4][4] = {{xx + yy + zz, yz - zy, zx - xz, xy - yx},
                              {yz - zy, xx - yy - zz, xy + yx, zx + xz},
                              {zx - xz, xy + yx, -xx + yy - zz, yz + zy},
                              {xy - yx, zx + xz, yz + zy, -xx - yy + zz}};
            jacobi4_top(K, q);
        }
        const double w = q[0], x = q[1], y = q[2], z = q[3];
        s_R[0] = w * w + x * x - y * y - z * z; s_R[1] = 2.0 * (x * y - w * z);         s_R[2] = 2.0 * (x * z + w * y);
        s_R[3] = 2.0 * (x * y + w * z);         s_R[4] = w * w - x * x + y * y - z * z; s_R[5] = 2.0 * (y * z - w * x);
        s_R[6] = 2.0 * (x * z - w * y);         s_R[7] = 2.0 * (y * z + w * x);         s_R[8] = w * w - x * x - y * y + z * z;
    }
    __syncthreads();
    double R[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = s_R[k];
    // pass 3: residual of the applied transform, and the superimposed coordinates R (b - cb) + ca
    double e = 0.0;
    for (int i = threadIdx.x; i < npts; i += kThreads) {
        double a[3], b[3], w;
        load(i, a, b, w);
        double y[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            y[r] = empty ? b[r] : R[3 * r] * (b[0] - cb[0]) + R[3 * r + 1] * (b[1] - cb[1]) + R[3 * r + 2] * (b[2] - cb[2]);
            const double d = y[r] - (a[r] - ca[r]);
            e += w * d * d;
        }
        if (o.coords) {
            double* dst = o.coords + (s * npts + i) * 3;
#pragma unroll
            for (int r = 0; r < 3; ++r) dst[r] = empty ? b[r] : y[r] + ca[r];
        }
    }
    e = block_sum(e, red);
    if (threadIdx.x == 0) {
        o.rmsd[s] = empty ? nan("") : sqrt(e / W);
        if (o.rot)
            for (int k = 0; k < 9; ++k) o.rot[9 * s + k] = R[k];
        if (o.trans)
            for (int r = 0; r < 3; ++r)
                o.trans[3 * s + r] = empty ? 0.0 : ca[r] - (R[3 * r] * cb[0] + R[3 * r + 1] * cb[1] + R[3 * r + 2] * cb[2]);
    }
}

// ------------------------------------------------------------------------------------------------------------
// dRMSD (validation_metrics.py:17-36): d_k[i][j] = |x_i - x_j| of each structure, sum (d1 - d2)^2 (m_i m_j) over the
// grid, n = min over sets of sum m (n = N without a mask), drmsd = sqrt(sum / (n (n - 1))) when n > 1, else sqrt(sum * 0).
// premul multiplies the coordinates by the mask first (compute_validation_metrics_all passes masked coordinates).
// Tile kernel: grid (T*T, B) with T = ceil(N / 64); partial[s][tile] is the tile's sum in a fixed order.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) drmsd_tile_kernel(const PointSets P, int N, int premul, double* __restrict__ partial) {
    __shared__ double red[kThreads];
    __shared__ double s_row[2][kTile][3], s_col[2][kTile][3], s_mr[kTile], s_mc[kTile];
    const int T = (N + kTile - 1) / kTile;
    const int ti = blockIdx.x / T, tj = blockIdx.x % T;
    const long s = blockIdx.y;
    for (int k = threadIdx.x; k < 2 * kTile; k += kThreads) {
        const bool col = k >= kTile;
        const int l = col ? k - kTile : k;
        const int i = (col ? tj : ti) * kTile + l;
        double m = 0.0, a[3] = {0.0, 0.0, 0.0}, b[3] = {0.0, 0.0, 0.0};
        if (i < N) {
            m = ld_mask(P, s, i);
            const long o = s * P.sstride + (long)i * P.pstride;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                a[c] = ldv(P.a, P.a64, o + c);
                b[c] = ldv(P.b, P.b64, o + c);
                if (premul) { a[c] *= m; b[c] *= m; }
            }
        }
        double (*dst)[kTile][3] = col ? s_col : s_row;
#pragma unroll
        for (int c = 0; c < 3; ++c) { dst[0][l][c] = a[c]; dst[1][l][c] = b[c]; }
        (col ? s_mc : s_mr)[l] = i < N ? m : 0.0;
    }
    __syncthreads();
    const int il = threadIdx.x % kTile;
    const int i = ti * kTile + il;
    double acc = 0.0;
    if (i < N) {
        for (int jl = threadIdx.x / kTile; jl < kTile; jl += kThreads / kTile) {
            if (tj * kTile + jl >= N) break;
            double d[2];
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                const double dx = s_row[k][il][0] - s_col[k][jl][0], dy = s_row[k][il][1] - s_col[k][jl][1],
                             dz = s_row[k][il][2] - s_col[k][jl][2];
                d[k] = sqrt(dx * dx + dy * dy + dz * dz);
            }
            const double dd = d[0] - d[1];
            acc += dd * dd * (s_mr[il] * s_mc[jl]);
        }
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) partial[s * (long)gridDim.x + blockIdx.x] = acc;
}

__global__ void __launch_bounds__(kThreads) drmsd_reduce_kernel(const PointSets P, int N, int B, int tiles,
                                                                const double* __restrict__ partial, double* __restrict__ out) {
    __shared__ double red[kThreads];
    double n = (double)N;
    if (P.m) {
        n = INFINITY;
        for (int s = 0; s < B; ++s) {
            double c = 0.0;
            for (int i = threadIdx.x; i < N; i += kThreads) c += ld_mask(P, s, i);
            n = fmin(n, block_sum(c, red));
        }
    }
    for (int s = 0; s < B; ++s) {
        double v = 0.0;
        for (int k = threadIdx.x; k < tiles; k += kThreads) v += partial[(long)s * tiles + k];
        v = block_sum(v, red);
        if (threadIdx.x == 0) out[s] = n > 1.0 ? sqrt(v * (1.0 / (n * (n - 1.0)))) : sqrt(v * 0.0);
    }
}

}  // namespace
}  // namespace dfold

using namespace dfold;

extern "C" int dfold_rot_trans_error(const void* pred, int pred_f64, const void* gt, int gt_f64, int nf, int N, int ref_frame,
                                     double* out, void* stream) {
    DFOLD_REQUIRE(pred && gt && out, "dfold_rot_trans_error: null pointer");
    DFOLD_REQUIRE(nf > 0 && N > 0, "dfold_rot_trans_error: need nf >= 1 and N >= 1 (got %d, %d)", nf, N);
    DFOLD_REQUIRE(ref_frame >= 0 && ref_frame < nf, "dfold_rot_trans_error: ref_frame %d outside [0, %d)", ref_frame, nf);
    rigid_error_kernel<<<(unsigned)nf, kThreads, 0, as_stream(stream)>>>(pred, pred_f64 != 0, gt, gt_f64 != 0, N, ref_frame, nf, out);
    return check_launch("rigid_error_kernel");
}

extern "C" int dfold_atom_errors(const void* pred, int pred_f64, const void* gt, int gt_f64, const void* mask, int mask_f64, int nf,
                                 int N, int A, int drop_last_atom, double* out, void* stream) {
    DFOLD_REQUIRE(pred && gt && mask && out, "dfold_atom_errors: null pointer");
    DFOLD_REQUIRE(nf > 0 && N > 0, "dfold_atom_errors: need nf >= 1 and N >= 1 (got %d, %d)", nf, N);
    DFOLD_REQUIRE(A >= 2, "dfold_atom_errors: A = %d, need A >= 2 (CA is atom column 1)", A);
    atom_error_kernel<<<(unsigned)nf, kThreads, 0, as_stream(stream)>>>(pred, pred_f64 != 0, gt, gt_f64 != 0, mask, mask_f64 != 0, N, A,
                                                                        drop_last_atom != 0, nf, out);
    return check_launch("atom_error_kernel");
}

extern "C" int dfold_superimpose(const void* reference, int reference_f64, const void* coords, int coords_f64, long set_stride,
                                 long point_stride, const void* mask, int mask_f64, long mask_set_stride, long mask_point_stride,
                                 int mask_mode, int B, int P, double* rmsd, double* rot, double* trans, double* out_coords,
                                 void* stream) {
    DFOLD_REQUIRE(reference && coords && rmsd, "dfold_superimpose: null pointer");
    DFOLD_REQUIRE(B > 0 && P > 0, "dfold_superimpose: need B >= 1 and P >= 1 (got %d, %d)", B, P);
    DFOLD_REQUIRE(set_stride >= 0 && point_stride >= 3, "dfold_superimpose: bad strides");
    DFOLD_REQUIRE(mask_mode >= 0 && mask_mode <= 2, "dfold_superimpose: mask_mode %d not in {0, 1, 2}", mask_mode);
    DFOLD_REQUIRE(mask_mode == 0 || mask, "dfold_superimpose: mask_mode %d needs a mask", mask_mode);
    PointSets ps{reference, reference_f64 != 0, coords, coords_f64 != 0, set_stride, point_stride,
                 mask_mode ? mask : nullptr, mask_f64 != 0, mask_set_stride, mask_point_stride};
    superimpose_kernel<<<(unsigned)B, kThreads, 0, as_stream(stream)>>>(ps, P, mask_mode, SupOut{rmsd, rot, trans, out_coords});
    return check_launch("superimpose_kernel");
}

extern "C" int dfold_drmsd(const void* s1, int s1_f64, const void* s2, int s2_f64, long set_stride, long point_stride,
                           const void* mask, int mask_f64, long mask_set_stride, long mask_point_stride, int premul, int B, int N,
                           double* partial, double* out, void* stream) {
    DFOLD_REQUIRE(s1 && s2 && partial && out, "dfold_drmsd: null pointer");
    DFOLD_REQUIRE(B > 0 && N > 0, "dfold_drmsd: need B >= 1 and N >= 1 (got %d, %d)", B, N);
    DFOLD_REQUIRE(B <= 65535, "dfold_drmsd: B = %d exceeds 65535 point sets", B);
    DFOLD_REQUIRE(set_stride >= 0 && point_stride >= 3, "dfold_drmsd: bad strides");
    DFOLD_REQUIRE(!premul || mask, "dfold_drmsd: premul needs a mask");
    const int T = (N + kTile - 1) / kTile;
    PointSets ps{s1, s1_f64 != 0, s2, s2_f64 != 0, set_stride, point_stride, mask, mask_f64 != 0, mask_set_stride, mask_point_stride};
    drmsd_tile_kernel<<<dim3((unsigned)(T * T), (unsigned)B), kThreads, 0, as_stream(stream)>>>(ps, N, premul != 0, partial);
    if (check_launch("drmsd_tile_kernel")) return 1;
    drmsd_reduce_kernel<<<1, kThreads, 0, as_stream(stream)>>>(ps, N, B, T * T, partial, out);
    return check_launch("drmsd_reduce_kernel");
}
