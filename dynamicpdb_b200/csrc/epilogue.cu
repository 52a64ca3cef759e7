// Epilogue kernels of the score network and the remaining rigid algebra (all 3x3 / quaternion math in registers).
//
//   score_fwd / score_bwd      K9: predicted frame + noised frame + t  ->  IGSO(3) rotation score (fp64 series, L terms)
//                              and VP-SDE translation score, one warp per residue, no [n,L] temporaries, sigma(t) looked
//                              up on the device.  Replaces (reference file:line) src/data/se3_diffuser.py:115-125,
//                              src/data/utils.py:589-606, src/data/so3_diffuser.py:9-49,71-117,274-305,
//                              src/data/r3_diffuser.py:42,169-177.
//   frames_to_atoms            K10: backbone frame o default frames o torsion rotations -> 8 rigid groups -> atom14 ->
//                              atom37, one warp per residue.  Replaces openfold/utils/feats.py:165-228,
//                              src/data/all_atom.py:114-154, src/model/Dfold_network_dynamic.py:574-594.
//   quat_mul, rot_compose      openfold/utils/rigid_utils.py:254-275 (quat_multiply, quat_multiply_by_vec), :22-106
//                              (rot_matmul, rot_vec_mul), :618-702 (Rotation.compose_r/apply/invert_apply),
//                              :1065-1146 (Rigid.compose / apply / invert_apply / invert) and their autograd.
#include "common.cuh"
#include "igso3.cuh"

namespace dfold {
namespace {

// ------------------------------------------------------------------------------------------------------------
// quaternion helpers (w, x, y, z)
// ------------------------------------------------------------------------------------------------------------
struct Q4 { float w, x, y, z; };
__device__ __forceinline__ Q4 qmul(const Q4& a, const Q4& b) {
    return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z,
            a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x,
            a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w};
}
__device__ __forceinline__ Q4 qconj(const Q4& a) { return {a.w, -a.x, -a.y, -a.z}; }
__device__ __forceinline__ Q4 ldq(const float* p) {
    const float4 v = *reinterpret_cast<const float4*>(p);
    return {v.x, v.y, v.z, v.w};
}

// ------------------------------------------------------------------------------------------------------------
// K9 score epilogue
// ------------------------------------------------------------------------------------------------------------
struct ScoreParams {
    const float* q_pred;     // [n,4] predicted rotation (rots_0 of calc_rot_score), any norm
    const float* q_t;        // [n,4] noised rotation (rots_t)
    const float* x_pred;     // [n,3] predicted translation BEFORE unscaling
    const float* x_t;        // [n,3] noised translation
    const double* t;         // device scalar
    const double* grid;      // [G] discrete sigma grid (so3_diffuser.discrete_sigma)
    int G;
    double e_max, e_min;     // exp(max_sigma), exp(min_sigma)
    double min_b, max_b;     // VP-SDE schedule
    float r3_scale;          // r3 coordinate_scaling (applied to both translations, r3_diffuser._scale)
    float inv_ipa_scale;     // 1 / ipa coordinate_scaling (the unscale of the predicted translation)
    const float* mask;       // [n] or null
    int L;
    long n;
};

__device__ __forceinline__ double sigma_of_t(const ScoreParams& p) {
    return p.grid[sigma_index(*p.t, p.grid, p.G, p.e_max, p.e_min)];
}

// everything between the two quaternions and the rotation vector, fp32 as in the reference (utils.py:589-606)
struct RotVec {
    Q4 q;            // q0t after the sign flip
    float sgn;       // +-1
    float nrm;       // |q.xyz|
    float angle, scale;
    int small;
    float vx, vy, vz;
    float vnorm;     // |vec|
};
__device__ __forceinline__ RotVec rotvec_of(const Q4& qp, const Q4& qt, Q4& inv, float& n2) {
    RotVec r;
    n2 = qp.w * qp.w + qp.x * qp.x + qp.y * qp.y + qp.z * qp.z;
    const Q4 c = qconj(qp);
    inv = {c.w / n2, c.x / n2, c.y / n2, c.z / n2};               // invert_quat, rigid_utils.py:282-286
    Q4 q = qmul(inv, qt);
    r.sgn = (q.w < 0.f) ? -1.f : 1.f;
    q = {q.w * r.sgn, q.x * r.sgn, q.y * r.sgn, q.z * r.sgn};
    r.q = q;
    r.nrm = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z);
    r.angle = 2.f * atan2f(r.nrm, q.w);
    const float a2 = r.angle * r.angle;
    r.small = r.angle <= 1e-3f;
    r.scale = r.small ? (2.f + a2 / 12.f + 7.f * a2 * a2 / 2880.f) : (r.angle / sinf(r.angle * 0.5f + 1e-6f));
    r.vx = r.scale * q.x; r.vy = r.scale * q.y; r.vz = r.scale * q.z;
    r.vnorm = sqrtf(r.vx * r.vx + r.vy * r.vy + r.vz * r.vz);
    return r;
}

template <typename TT>
__global__ void __launch_bounds__(256) score_fwd_kernel(const ScoreParams p, double* __restrict__ rot_score, TT* __restrict__ trans_score) {
    const long i = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= p.n) return;
    const int lane = threadIdx.x & 31;
    const float m = p.mask ? p.mask[i] : 1.f;
    if (rot_score) {
        const double sigma = sigma_of_t(p);
        Q4 inv; float n2;
        const RotVec r = rotvec_of(ldq(p.q_pred + 4 * i), ldq(p.q_t + 4 * i), inv, n2);
        const float omega = r.vnorm + 1e-6f;
        double S, dS, d2S;
        igso3_series<float, false>(omega, sigma, p.L, lane, S, dS, d2S);
        if (lane < 3) {
            const double g = dS / (S + 1e-4);
            const float v = lane == 0 ? r.vx : (lane == 1 ? r.vy : r.vz);
            rot_score[3 * i + lane] = g * (double)v / (double)(omega + 1e-6f) * (double)m;
        }
    }
    if (trans_score && lane < 3) {
        const double t = *p.t;
        const double beta = t * p.min_b + 0.5 * t * t * (p.max_b - p.min_b);
        const float a = p.x_t[3 * i + lane] * p.r3_scale;
        const float b = (p.x_pred[3 * i + lane] * p.inv_ipa_scale) * p.r3_scale;
        const double sc = -((double)a - exp(-0.5 * beta) * (double)b) / (1.0 - exp(-beta));
        trans_score[3 * i + lane] = (TT)(sc * (double)m);
    }
}

template <typename TT>
__global__ void __launch_bounds__(256) score_bwd_kernel(const ScoreParams p, const double* __restrict__ d_rot, const TT* __restrict__ d_trans,
                                                        float* __restrict__ dq_pred, float* __restrict__ dx_pred) {
    const long i = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= p.n) return;
    const int lane = threadIdx.x & 31;
    const float m = p.mask ? p.mask[i] : 1.f;
    if (dq_pred) {
        if (d_rot == nullptr) {
            if (lane < 4) dq_pred[4 * i + lane] = 0.f;
        } else {
            const double sigma = sigma_of_t(p);
            const Q4 qp = ldq(p.q_pred + 4 * i), qt = ldq(p.q_t + 4 * i);
            Q4 inv; float n2;
            const RotVec r = rotvec_of(qp, qt, inv, n2);
            const float omega = r.vnorm + 1e-6f;
            double S, dS, d2S;
            igso3_series<float, true>(omega, sigma, p.L, lane, S, dS, d2S);
            if (lane == 0) {
                const double den = S + 1e-4;
                const double g = dS / den;
                const double gp = d2S / den - dS * dS / (den * den);
                const double om_e = (double)(omega + 1e-6f);
                const double c = g / om_e;
                const double dc_dom = gp / om_e - g / (om_e * om_e);
                const double gx = d_rot[3 * i] * m, gy = d_rot[3 * i + 1] * m, gz = d_rot[3 * i + 2] * m;
                // score = c * vec
                double dvx = c * gx, dvy = c * gy, dvz = c * gz;
                const double dcoef = gx * r.vx + gy * r.vy + gz * r.vz;
                const double dom = dcoef * dc_dom;
                if (r.vnorm > 0.f) {
                    const double k = dom / (double)r.vnorm;
                    dvx += k * r.vx; dvy += k * r.vy; dvz += k * r.vz;
                }
                // vec = scale * q.xyz
                const double dscale = dvx * r.q.x + dvy * r.q.y + dvz * r.q.z;
                double dqx = r.scale * dvx, dqy = r.scale * dvy, dqz = r.scale * dvz, dqw = 0.0;
                double ds_da;
                const double a = r.angle;
                if (r.small) {
                    ds_da = a / 6.0 + 7.0 * a * a * a / 720.0;
                } else {
                    const double sn = sin(a * 0.5 + 1e-6), cs = cos(a * 0.5 + 1e-6);
                    ds_da = 1.0 / sn - a * 0.5 * cs / (sn * sn);
                }
                const double dangle = dscale * ds_da;
                // angle = 2 atan2(nrm, w)
                const double den2 = (double)r.nrm * r.nrm + (double)r.q.w * r.q.w;
                if (den2 > 0.0) {
                    const double dn = 2.0 * r.q.w / den2 * dangle;
                    dqw += -2.0 * r.nrm / den2 * dangle;
                    if (r.nrm > 0.f) {
                        const double k = dn / (double)r.nrm;
                        dqx += k * r.q.x; dqy += k * r.q.y; dqz += k * r.q.z;
                    }
                }
                // undo the sign flip, then q0t = inv (x) qt  ->  d inv = d q0t (x) conj(qt)
                const Q4 d0t = {(float)(dqw * r.sgn), (float)(dqx * r.sgn), (float)(dqy * r.sgn), (float)(dqz * r.sgn)};
                const Q4 dinv = qmul(d0t, qconj(qt));
                // inv = conj(qp) / n2
                const Q4 cj = qconj(qp);
                const float dn2 = -(dinv.w * cj.w + dinv.x * cj.x + dinv.y * cj.y + dinv.z * cj.z) / (n2 * n2);
                float4 o;
                o.x = dinv.w / n2 + 2.f * qp.w * dn2;
                o.y = -dinv.x / n2 + 2.f * qp.x * dn2;
                o.z = -dinv.y / n2 + 2.f * qp.y * dn2;
                o.w = -dinv.z / n2 + 2.f * qp.z * dn2;
                *reinterpret_cast<float4*>(dq_pred + 4 * i) = o;
            }
        }
    }
    if (dx_pred && lane < 3) {
        float g = 0.f;
        if (d_trans) {
            const double t = *p.t;
            const double beta = t * p.min_b + 0.5 * t * t * (p.max_b - p.min_b);
            // score = -(a - E b) / D,  b = x_pred * inv_ipa * r3  ->  d/dx_pred = E * inv_ipa * r3 / D
            g = (float)((double)d_trans[3 * i + lane] * (double)m * exp(-0.5 * beta) / (1.0 - exp(-beta))
                        * (double)p.inv_ipa_scale * (double)p.r3_scale);
        }
        dx_pred[3 * i + lane] = g;
    }
}

// ------------------------------------------------------------------------------------------------------------
// K10 frames -> atoms
// ------------------------------------------------------------------------------------------------------------
struct Fr { float R[9]; float t[3]; };
__device__ __forceinline__ Fr fr_compose(const Fr& a, const Fr& b) {          // a o b  (Rigid.compose, rigid_utils.py:1065-1079)
    Fr o;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
        for (int c = 0; c < 3; ++c) o.R[3 * r + c] = a.R[3 * r] * b.R[c] + a.R[3 * r + 1] * b.R[3 + c] + a.R[3 * r + 2] * b.R[6 + c];
        o.t[r] = a.R[3 * r] * b.t[0] + a.R[3 * r + 1] * b.t[1] + a.R[3 * r + 2] * b.t[2] + a.t[r];
    }
    return o;
}

struct AtomTables {
    const float* default_frames;    // [21,8,4,4]
    const long* atom14_group;       // [21,14]
    const float* atom14_mask;       // [21,14]
    const float* atom14_pos;        // [21,14,3]
    const long* atom37_to_atom14;   // [21,37]
    const float* atom37_mask;       // [21,37]
};

// rot_mode 0: backbone rotation given as quaternion [n,4]; 1: as row-major 3x3 [n,9]
__global__ void __launch_bounds__(256) frames_to_atoms_kernel(const float* __restrict__ rot, int rot_mode, const float* __restrict__ trans,
                                                              const float* __restrict__ alpha, const long* __restrict__ aatype,
                                                              const AtomTables tb, float* __restrict__ frames44, float* __restrict__ atom14,
                                                              float* __restrict__ atom37, long n) {
    __shared__ float s_fr[8][8][12];     // [warp][group][R(9) t(3)]
    __shared__ float s_a14[8][14][3];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long i = (long)blockIdx.x * 8 + wib;
    if (i >= n) return;
    const int aa = (int)aatype[i];
    // ---- group frames: default_g o Rx(alpha_g); group 0 has the identity torsion (feats.py:184-207) ----
    if (lane < 8) {
        const float* d = tb.default_frames + ((long)aa * 8 + lane) * 16;
        float sn = 0.f, cs = 1.f;
        if (lane > 0) { sn = alpha[(i * 7 + lane - 1) * 2]; cs = alpha[(i * 7 + lane - 1) * 2 + 1]; }
        // R = Rd * [[1,0,0],[0,c,-s],[0,s,c]]
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float d0 = d[4 * r], d1 = d[4 * r + 1], d2 = d[4 * r + 2];
            s_fr[wib][lane][3 * r] = d0;
            s_fr[wib][lane][3 * r + 1] = d1 * cs + d2 * sn;
            s_fr[wib][lane][3 * r + 2] = -d1 * sn + d2 * cs;
            s_fr[wib][lane][9 + r] = d[4 * r + 3];
        }
    }
    __syncwarp();
    // ---- chi chain: chi2 = chi1 o f5, chi3 = chi2 o f6, chi4 = chi3 o f7 (feats.py:209-213) ----
    if (lane == 0) {
        Fr acc;
#pragma unroll
        for (int k = 0; k < 12; ++k) (k < 9 ? acc.R[k] : acc.t[k - 9]) = s_fr[wib][4][k];
        for (int g = 5; g < 8; ++g) {
            Fr b;
#pragma unroll
            for (int k = 0; k < 12; ++k) (k < 9 ? b.R[k] : b.t[k - 9]) = s_fr[wib][g][k];
            acc = fr_compose(acc, b);
#pragma unroll
            for (int k = 0; k < 12; ++k) s_fr[wib][g][k] = (k < 9 ? acc.R[k] : acc.t[k - 9]);
        }
    }
    __syncwarp();
    // ---- to global: backbone o group (feats.py:226) ----
    if (lane < 8) {
        Fr bb;
        if (rot_mode == 0) {
            const Q4 q = ldq(rot + 4 * i);
            quat_to_rot9(q.w, q.x, q.y, q.z, bb.R);
        } else {
#pragma unroll
            for (int k = 0; k < 9; ++k) bb.R[k] = rot[9 * i + k];
        }
        bb.t[0] = trans[3 * i]; bb.t[1] = trans[3 * i + 1]; bb.t[2] = trans[3 * i + 2];
        Fr g;
#pragma unroll
        for (int k = 0; k < 12; ++k) (k < 9 ? g.R[k] : g.t[k - 9]) = s_fr[wib][lane][k];
        const Fr o = fr_compose(bb, g);
#pragma unroll
        for (int k = 0; k < 12; ++k) s_fr[wib][lane][k] = (k < 9 ? o.R[k] : o.t[k - 9]);
        if (frames44) {
            float* f = frames44 + (i * 8 + lane) * 16;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                f[4 * r] = o.R[3 * r]; f[4 * r + 1] = o.R[3 * r + 1]; f[4 * r + 2] = o.R[3 * r + 2]; f[4 * r + 3] = o.t[r];
            }
            f[12] = 0.f; f[13] = 0.f; f[14] = 0.f; f[15] = 1.f;
        }
    }
    __syncwarp();
    // ---- atom14 = frame[group(atom)] applied to the idealised position, masked (all_atom.py:129-154) ----
    if (lane < 14) {
        const int g = (int)tb.atom14_group[aa * 14 + lane];
        const float* lit = tb.atom14_pos + ((long)aa * 14 + lane) * 3;
        const float mk = tb.atom14_mask[aa * 14 + lane];
        const float* fr = s_fr[wib][g];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const float v = (fr[3 * r] * lit[0] + fr[3 * r + 1] * lit[1] + fr[3 * r + 2] * lit[2] + fr[9 + r]) * mk;
            s_a14[wib][lane][r] = v;
        }
    }
    __syncwarp();
    if (atom14)
        for (int k = lane; k < 42; k += 32) atom14[i * 42 + k] = s_a14[wib][k / 3][k % 3];
    if (atom37)
        for (int k = lane; k < 111; k += 32) {
            const int a = k / 3;
            const int src = (int)tb.atom37_to_atom14[aa * 37 + a];
            atom37[i * 111 + k] = s_a14[wib][src][k % 3] * tb.atom37_mask[aa * 37 + a];
        }
}

// ------------------------------------------------------------------------------------------------------------
// quaternion product / rotation-matrix composition with autograd
// ------------------------------------------------------------------------------------------------------------
// out = a (x) b ; b is a quaternion [n,4] or (b_is_vec) a pure vector [n,3] = (0, v)
__global__ void quat_mul_fwd_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, long n, int b_is_vec) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Q4 qa = ldq(a + 4 * i);
    const Q4 qb = b_is_vec ? Q4{0.f, b[3 * i], b[3 * i + 1], b[3 * i + 2]} : ldq(b + 4 * i);
    const Q4 o = qmul(qa, qb);
    *reinterpret_cast<float4*>(out + 4 * i) = make_float4(o.w, o.x, o.y, o.z);
}
// <g, a b> = <g b*, a> = <a* g, b>
__global__ void quat_mul_bwd_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ g,
                                    float* __restrict__ da, float* __restrict__ db, long n, int b_is_vec) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Q4 qa = ldq(a + 4 * i);
    const Q4 qb = b_is_vec ? Q4{0.f, b[3 * i], b[3 * i + 1], b[3 * i + 2]} : ldq(b + 4 * i);
    const Q4 gg = ldq(g + 4 * i);
    if (da) {
        const Q4 o = qmul(gg, qconj(qb));
        *reinterpret_cast<float4*>(da + 4 * i) = make_float4(o.w, o.x, o.y, o.z);
    }
    if (db) {
        const Q4 o = qmul(qconj(qa), gg);
        if (b_is_vec) { db[3 * i] = o.x; db[3 * i + 1] = o.y; db[3 * i + 2] = o.z; }
        else *reinterpret_cast<float4*>(db + 4 * i) = make_float4(o.w, o.x, o.y, o.z);
    }
}

// One thread per LEFT frame a (na of them); it serves `rep` consecutive right operands b (trailing broadcast of a).
//   Rout = Ra Rb                      (when Rb given)
//   tout = Ra tb + ta                 (when tb given; ta optional)         inverse: tout = Ra^T (tb - ta)
__global__ void rot_compose_fwd_kernel(const float* __restrict__ Ra, const float* __restrict__ ta, const float* __restrict__ Rb,
                                       const float* __restrict__ tb, float* __restrict__ Rout, float* __restrict__ tout,
                                       long na, int rep, int inverse) {
    const long ia = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (ia >= na) return;
    float A[9], at[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 9; ++k) A[k] = Ra[9 * ia + k];
    if (ta) { at[0] = ta[3 * ia]; at[1] = ta[3 * ia + 1]; at[2] = ta[3 * ia + 2]; }
    for (int j = 0; j < rep; ++j) {
        const long ib = ia * rep + j;
        if (Rb && Rout) {
            float B[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) B[k] = Rb[9 * ib + k];
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    Rout[9 * ib + 3 * r + c] = A[3 * r] * B[c] + A[3 * r + 1] * B[3 + c] + A[3 * r + 2] * B[6 + c];
        }
        if (tb && tout) {
            float x = tb[3 * ib], y = tb[3 * ib + 1], z = tb[3 * ib + 2];
            if (!inverse) {
#pragma unroll
                for (int r = 0; r < 3; ++r) tout[3 * ib + r] = A[3 * r] * x + A[3 * r + 1] * y + A[3 * r + 2] * z + at[r];
            } else {
                x -= at[0]; y -= at[1]; z -= at[2];
#pragma unroll
                for (int r = 0; r < 3; ++r) tout[3 * ib + r] = A[r] * x + A[3 + r] * y + A[6 + r] * z;
            }
        }
    }
}

__global__ void rot_compose_bwd_kernel(const float* __restrict__ Ra, const float* __restrict__ ta, const float* __restrict__ Rb,
                                       const float* __restrict__ tb, const float* __restrict__ dRout, const float* __restrict__ dtout,
                                       float* __restrict__ dRa, float* __restrict__ dta, float* __restrict__ dRb, float* __restrict__ dtb,
                                       long na, int rep, int inverse) {
    const long ia = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (ia >= na) return;
    float A[9], at[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 9; ++k) A[k] = Ra[9 * ia + k];
    if (ta) { at[0] = ta[3 * ia]; at[1] = ta[3 * ia + 1]; at[2] = ta[3 * ia + 2]; }
    float gA[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, gat[3] = {0.f, 0.f, 0.f};
    for (int j = 0; j < rep; ++j) {
        const long ib = ia * rep + j;
        if (Rb && dRout) {
            float B[9], G[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) { B[k] = Rb[9 * ib + k]; G[k] = dRout[9 * ib + k]; }
            // dA = G B^T ; dB = A^T G
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    gA[3 * r + c] += G[3 * r] * B[3 * c] + G[3 * r + 1] * B[3 * c + 1] + G[3 * r + 2] * B[3 * c + 2];
                    if (dRb) dRb[9 * ib + 3 * r + c] = A[r] * G[c] + A[3 + r] * G[3 + c] + A[6 + r] * G[6 + c];
                }
        } else if (dRb) {
#pragma unroll
            for (int k = 0; k < 9; ++k) dRb[9 * ib + k] = 0.f;
        }
        if (tb && dtout) {
            const float g0 = dtout[3 * ib], g1 = dtout[3 * ib + 1], g2 = dtout[3 * ib + 2];
            float x = tb[3 * ib], y = tb[3 * ib + 1], z = tb[3 * ib + 2];
            if (!inverse) {
                // tout = A x + at
                const float g[3] = {g0, g1, g2};
#pragma unroll
                for (int r = 0; r < 3; ++r) {
                    gA[3 * r] += g[r] * x; gA[3 * r + 1] += g[r] * y; gA[3 * r + 2] += g[r] * z;
                    gat[r] += g[r];
                }
                if (dtb) {
#pragma unroll
                    for (int c = 0; c < 3; ++c) dtb[3 * ib + c] = A[c] * g0 + A[3 + c] * g1 + A[6 + c] * g2;
                }
            } else {
                // tout = A^T (x - at):  tout_r = sum_k A[k][r] (x_k - at_k)
                x -= at[0]; y -= at[1]; z -= at[2];
                const float d[3] = {x, y, z}, g[3] = {g0, g1, g2};
#pragma unroll
                for (int k = 0; k < 3; ++k)
#pragma unroll
                    for (int r = 0; r < 3; ++r) gA[3 * k + r] += d[k] * g[r];
                float dx[3];
#pragma unroll
                for (int k = 0; k < 3; ++k) dx[k] = A[3 * k] * g0 + A[3 * k + 1] * g1 + A[3 * k + 2] * g2;
                if (dtb) { dtb[3 * ib] = dx[0]; dtb[3 * ib + 1] = dx[1]; dtb[3 * ib + 2] = dx[2]; }
                gat[0] -= dx[0]; gat[1] -= dx[1]; gat[2] -= dx[2];
            }
        } else if (dtb) {
            dtb[3 * ib] = 0.f; dtb[3 * ib + 1] = 0.f; dtb[3 * ib + 2] = 0.f;
        }
    }
    if (dRa) {
#pragma unroll
        for (int k = 0; k < 9; ++k) dRa[9 * ia + k] = gA[k];
    }
    if (dta) { dta[3 * ia] = gat[0]; dta[3 * ia + 1] = gat[1]; dta[3 * ia + 2] = gat[2]; }
}


// ------------------------------------------------------------------------------------------------------------
// reverse-diffusion step (f2): one block per trajectory frame.  Replaces src/data/se3_diffuser.py:160-215,
// so3_diffuser.py:329-365 (geodesic random walk, right multiplication), r3_diffuser.py:106-157 (VP-SDE Euler-Maruyama
// step + centring) and the scipy rotation-vector round trips (se3_diffuser.py:11-29); the noise is an input.
// ------------------------------------------------------------------------------------------------------------
struct ReverseParams {
    const float* q_t; const float* x_t;          // [F,N,4], [F,N,3]
    const double* rot_score; const void* trans_score; int trans_is_f64;
    const float* z_rot; const float* z_trans;    // N(0,1) draws [F,N,3] (already multiplied by noise_scale or not: see noise_scale)
    const float* mask;                           // diffuse mask [F,N] or null
    double g_rot, g_trans, b_t, dt, noise_scale, r3_scale;
    int center, diffuse_rot, diffuse_trans;
    float* q_out; float* x_out;
    int N;
};

__global__ void __launch_bounds__(256) reverse_step_kernel(const ReverseParams p) {
    __shared__ double s_sum[3][8];
    __shared__ double s_com[3];
    const int f = blockIdx.x;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long base = (long)f * p.N;
    const double sdt = sqrt(p.dt);
    double cx = 0.0, cy = 0.0, cz = 0.0;
    // pass 1: translations after the step (scaled units), accumulate the centre of mass
    for (int i = threadIdx.x; i < p.N; i += blockDim.x) {
        const long r = base + i;
        if (p.diffuse_trans) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const double x = (double)p.x_t[3 * r + c] * p.r3_scale;
                const double sc = p.trans_is_f64 ? ((const double*)p.trans_score)[3 * r + c] : (double)((const float*)p.trans_score)[3 * r + c];
                const double z = p.noise_scale * (double)p.z_trans[3 * r + c];
                const double perturb = (-0.5 * p.b_t * x - p.g_trans * p.g_trans * sc) * p.dt + p.g_trans * sdt * z;
                const double x1 = x - perturb;
                (c == 0 ? cx : (c == 1 ? cy : cz)) += x1;
            }
        }
    }
    if (p.diffuse_trans && p.center) {
        cx = warp_sum_d(cx); cy = warp_sum_d(cy); cz = warp_sum_d(cz);
        if (lane == 0) { s_sum[0][wid] = cx; s_sum[1][wid] = cy; s_sum[2][wid] = cz; }
        __syncthreads();
        if (threadIdx.x < 3) {
            double t = 0.0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_sum[threadIdx.x][w];
            s_com[threadIdx.x] = t / (double)p.N;             // r3_diffuser.py:151 with the default all-ones mask
        }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < p.N; i += blockDim.x) {
        const long r = base + i;
        const bool upd = p.mask ? (p.mask[r] > 0.5f) : true;    // _apply_mask with a 0/1 mask (se3_diffuser.py:206-210)
        // ---- translation ----
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float out = p.x_t[3 * r + c];
            if (p.diffuse_trans && upd) {
                const double x = (double)p.x_t[3 * r + c] * p.r3_scale;
                const double sc = p.trans_is_f64 ? ((const double*)p.trans_score)[3 * r + c] : (double)((const float*)p.trans_score)[3 * r + c];
                const double z = p.noise_scale * (double)p.z_trans[3 * r + c];
                const double perturb = (-0.5 * p.b_t * x - p.g_trans * p.g_trans * sc) * p.dt + p.g_trans * sdt * z;
                double x1 = x - perturb;
                if (p.center) x1 -= s_com[c];
                out = (float)(x1 / p.r3_scale);
            }
            p.x_out[3 * r + c] = out;
        }
        // ---- rotation: R_{t-1} = R_t Exp(perturb)  <=>  q_{t-1} = q_t (x) (cos(a/2), sin(a/2) axis) ----
        const float4 q4 = *reinterpret_cast<const float4*>(p.q_t + 4 * r);
        double qw = q4.x, qx = q4.y, qy = q4.z, qz = q4.w;
        const double qn = sqrt(qw * qw + qx * qx + qy * qy + qz * qz);
        qw /= qn; qx /= qn; qy /= qn; qz /= qn;
        if (p.diffuse_rot && upd) {
            double v[3];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const double z = p.noise_scale * (double)p.z_rot[3 * r + c];
                v[c] = p.g_rot * p.g_rot * p.rot_score[3 * r + c] * p.dt + p.g_rot * sdt * z;
            }
            const double a = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
            double pw = 1.0, k = 0.5;                       // sin(a/2)/a -> 1/2
            if (a > 1e-12) { pw = cos(0.5 * a); k = sin(0.5 * a) / a; }
            const double px = k * v[0], py = k * v[1], pz = k * v[2];
            const double nw = qw * pw - qx * px - qy * py - qz * pz;
            const double nx = qw * px + qx * pw + qy * pz - qz * py;
            const double ny = qw * py - qx * pz + qy * pw + qz * px;
            const double nz = qw * pz + qx * py - qy * px + qz * pw;
            const double nn = sqrt(nw * nw + nx * nx + ny * ny + nz * nz);
            qw = nw / nn; qx = nx / nn; qy = ny / nn; qz = nz / nn;
        }
        *reinterpret_cast<float4*>(p.q_out + 4 * r) = make_float4((float)qw, (float)qx, (float)qy, (float)qz);
    }
}

int fill_score_params(ScoreParams& p, const float* q_pred, const float* q_t, const float* x_pred, const float* x_t, const double* t,
                      const double* grid, int G, double max_sigma, double min_sigma, double min_b, double max_b, float r3_scale,
                      float ipa_scale, const float* mask, int L, long n) {
    DFOLD_REQUIRE(n > 0 && L > 0 && G > 0, "dfold_score: empty problem");
    DFOLD_REQUIRE(t != nullptr && grid != nullptr, "dfold_score: t / sigma grid missing");
    DFOLD_REQUIRE(ipa_scale != 0.f, "dfold_score: zero coordinate scaling");
    p.q_pred = q_pred; p.q_t = q_t; p.x_pred = x_pred; p.x_t = x_t; p.t = t; p.grid = grid; p.G = G;
    p.e_max = exp(max_sigma); p.e_min = exp(min_sigma); p.min_b = min_b; p.max_b = max_b;
    p.r3_scale = r3_scale; p.inv_ipa_scale = 1.f / ipa_scale; p.mask = mask; p.L = L; p.n = n;
    return 0;
}

}  // namespace
}  // namespace dfold

using namespace dfold;

extern "C" int dfold_score_fwd(const float* q_pred, const float* q_t, const float* x_pred, const float* x_t, const double* t,
                               const double* sigma_grid, int G, double max_sigma, double min_sigma, double min_b, double max_b,
                               float r3_scale, float ipa_scale, const float* mask, int L, long n,
                               double* rot_score, void* trans_score, int trans_is_f64, void* stream) {
    ScoreParams p;
    if (fill_score_params(p, q_pred, q_t, x_pred, x_t, t, sigma_grid, G, max_sigma, min_sigma, min_b, max_b, r3_scale, ipa_scale, mask, L, n)) return 1;
    DFOLD_REQUIRE(rot_score == nullptr || (q_pred && q_t), "dfold_score_fwd: rotations missing");
    DFOLD_REQUIRE(trans_score == nullptr || (x_pred && x_t), "dfold_score_fwd: translations missing");
    const unsigned grid = (unsigned)cdiv(n, 8);
    if (trans_is_f64) score_fwd_kernel<double><<<grid, 256, 0, as_stream(stream)>>>(p, rot_score, (double*)trans_score);
    else score_fwd_kernel<float><<<grid, 256, 0, as_stream(stream)>>>(p, rot_score, (float*)trans_score);
    return check_launch("score_fwd_kernel");
}

extern "C" int dfold_score_bwd(const float* q_pred, const float* q_t, const float* x_pred, const float* x_t, const double* t,
                               const double* sigma_grid, int G, double max_sigma, double min_sigma, double min_b, double max_b,
                               float r3_scale, float ipa_scale, const float* mask, int L, long n,
                               const double* d_rot_score, const void* d_trans_score, int trans_is_f64,
                               float* dq_pred, float* dx_pred, void* stream) {
    ScoreParams p;
    if (fill_score_params(p, q_pred, q_t, x_pred, x_t, t, sigma_grid, G, max_sigma, min_sigma, min_b, max_b, r3_scale, ipa_scale, mask, L, n)) return 1;
    const unsigned grid = (unsigned)cdiv(n, 8);
    if (trans_is_f64) score_bwd_kernel<double><<<grid, 256, 0, as_stream(stream)>>>(p, d_rot_score, (const double*)d_trans_score, dq_pred, dx_pred);
    else score_bwd_kernel<float><<<grid, 256, 0, as_stream(stream)>>>(p, d_rot_score, (const float*)d_trans_score, dq_pred, dx_pred);
    return check_launch("score_bwd_kernel");
}

extern "C" int dfold_frames_to_atoms_fwd(const float* rot, int rot_is_matrix, const float* trans, const float* alpha, const long* aatype,
                                         const float* default_frames, const long* atom14_group, const float* atom14_mask,
                                         const float* atom14_pos, const long* atom37_to_atom14, const float* atom37_mask,
                                         float* frames44, float* atom14, float* atom37, long n, void* stream) {
    DFOLD_REQUIRE(n > 0, "dfold_frames_to_atoms_fwd: empty input");
    DFOLD_REQUIRE(rot && trans && alpha && aatype && default_frames && atom14_group && atom14_mask && atom14_pos,
                  "dfold_frames_to_atoms_fwd: null input");
    DFOLD_REQUIRE(atom37 == nullptr || (atom37_to_atom14 && atom37_mask), "dfold_frames_to_atoms_fwd: atom37 tables missing");
    AtomTables tb{default_frames, atom14_group, atom14_mask, atom14_pos, atom37_to_atom14, atom37_mask};
    frames_to_atoms_kernel<<<(unsigned)cdiv(n, 8), 256, 0, as_stream(stream)>>>(rot, rot_is_matrix, trans, alpha, aatype, tb, frames44,
                                                                                atom14, atom37, n);
    return check_launch("frames_to_atoms_kernel");
}

extern "C" int dfold_quat_mul_fwd(const float* a, const float* b, float* out, long n, int b_is_vec, void* stream) {
    DFOLD_REQUIRE(n > 0, "dfold_quat_mul_fwd: empty input");
    quat_mul_fwd_kernel<<<(unsigned)cdiv(n, 256), 256, 0, as_stream(stream)>>>(a, b, out, n, b_is_vec);
    return check_launch("quat_mul_fwd_kernel");
}
extern "C" int dfold_quat_mul_bwd(const float* a, const float* b, const float* dout, float* da, float* db, long n, int b_is_vec, void* stream) {
    DFOLD_REQUIRE(n > 0, "dfold_quat_mul_bwd: empty input");
    quat_mul_bwd_kernel<<<(unsigned)cdiv(n, 256), 256, 0, as_stream(stream)>>>(a, b, dout, da, db, n, b_is_vec);
    return check_launch("quat_mul_bwd_kernel");
}
extern "C" int dfold_rot_compose_fwd(const float* rot_a, const float* trans_a, const float* rot_b, const float* trans_b,
                                     float* rot_out, float* trans_out, long n_a, int rep, int inverse, void* stream) {
    DFOLD_REQUIRE(n_a > 0 && rep > 0 && rot_a, "dfold_rot_compose_fwd: empty input");
    rot_compose_fwd_kernel<<<(unsigned)cdiv(n_a, 128), 128, 0, as_stream(stream)>>>(rot_a, trans_a, rot_b, trans_b, rot_out, trans_out, n_a, rep, inverse);
    return check_launch("rot_compose_fwd_kernel");
}
extern "C" int dfold_rot_compose_bwd(const float* rot_a, const float* trans_a, const float* rot_b, const float* trans_b,
                                     const float* drot_out, const float* dtrans_out, float* drot_a, float* dtrans_a,
                                     float* drot_b, float* dtrans_b, long n_a, int rep, int inverse, void* stream) {
    DFOLD_REQUIRE(n_a > 0 && rep > 0 && rot_a, "dfold_rot_compose_bwd: empty input");
    rot_compose_bwd_kernel<<<(unsigned)cdiv(n_a, 128), 128, 0, as_stream(stream)>>>(rot_a, trans_a, rot_b, trans_b, drot_out, dtrans_out,
                                                                                   drot_a, dtrans_a, drot_b, dtrans_b, n_a, rep, inverse);
    return check_launch("rot_compose_bwd_kernel");
}

extern "C" int dfold_reverse_step(const float* q_t, const float* x_t, const double* rot_score, const void* trans_score, int trans_is_f64,
                                  const float* z_rot, const float* z_trans, const float* mask, double g_rot, double g_trans, double b_t,
                                  double dt, double noise_scale, double r3_scale, int center, int diffuse_rot, int diffuse_trans,
                                  float* q_out, float* x_out, long F, long N, void* stream) {
    DFOLD_REQUIRE(F > 0 && N > 0, "dfold_reverse_step: empty input");
    DFOLD_REQUIRE(q_t && x_t && q_out && x_out, "dfold_reverse_step: null frames");
    DFOLD_REQUIRE(!diffuse_rot || (rot_score && z_rot), "dfold_reverse_step: rotation score / noise missing");
    DFOLD_REQUIRE(!diffuse_trans || (trans_score && z_trans), "dfold_reverse_step: translation score / noise missing");
    ReverseParams p{q_t, x_t, rot_score, trans_score, trans_is_f64, z_rot, z_trans, mask, g_rot, g_trans, b_t, dt, noise_scale, r3_scale,
                    center, diffuse_rot, diffuse_trans, q_out, x_out, (int)N};
    reverse_step_kernel<<<(unsigned)F, 256, 0, as_stream(stream)>>>(p);
    return check_launch("reverse_step_kernel");
}
