// Training loss of the DFOLDv2 score network (SURVEY.md §8 f3), one kernel for value and gradients.
//
// Only the last trajectory frame is trained on (reference train_DFOLD_dynamics.py:1222, :1248, :1312), so the loss is a
// reduction over the N residues of that frame: torsion term (openfold/utils/loss.py:52-76, masked, an_weight = 0),
// rotation-score term (:1283-1305, or the axis / angle form :1255-1282), x0 translation term (:1248), the `< 100` gates
// (:1337-1339) and the normalisation by the number of non-empty frames (:1374-1375).  One CTA, fp64 throughout (the
// reference's loader hands float64 targets, which promotes the whole expression), deterministic tree reductions.
// The O((5N)^2) pair-distance tensors and the ground-truth backbone of :1316-1365 never reach final_loss and are not built.
// Gradients follow torch's autograd at the non-smooth points too: a vector norm has gradient 0 at 0, so a zero-length
// predicted torsion (sin, cos) keeps the direct term w / 1e-8 of u / (|u| + 1e-8), and a zero rotation score of a counted
// residue keeps d axis / 1e-6 of the separate loss's axis term; torch.minimum splits a tie between the two torsion
// targets evenly.
#include "common.cuh"

namespace dfold {
namespace {

constexpr int LT = 256;

__device__ double block_sum(double v, double* red) {
    v = warp_sum_d(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < LT / 32; ++w) t += red[w];
    return t;
}

struct LossParams {
    const double* ang;      // [N,7,2] predicted (normalised) torsion sin/cos of the last frame
    const double* a_gt; const double* a_alt; const double* a_mask;   // [N,7,2], [N,7,2], [N,7]
    const double* rs;       // [N,3]  predicted rotation score
    const double* gt_rot;   // [N,3]
    const double* x; const double* x0;      // [N,3] predicted / ground-truth translation
    const double* res_mask; const double* fixed_mask;   // [nf,N] (all frames: the normaliser counts non-empty frames)
    const double* t; const double* rot_scaling;         // device scalars
    int nf, N;
    double w_tor, w_rot, w_trans, t_thr;
    int rot_on, separate;
    double* out;            // [8]: loss, rot, trans, torsion (normalised), rot, trans, torsion, final (per frame)
    double* d_ang; double* d_rs; double* d_x;           // d loss / d input
};

__global__ void __launch_bounds__(LT) loss_kernel(const LossParams p) {
    __shared__ double red[LT / 32];
    const int N = p.N, tid = threadIdx.x;
    const double* rm = p.res_mask + (long)(p.nf - 1) * N;
    const double* fm = p.fixed_mask + (long)(p.nf - 1) * N;
    // ---- reductions ----
    double s_lm = 0, s_rot = 0, s_axis = 0, s_trans = 0, s_tor = 0, s_tm = 0, s_cnt = 0;
    const double scal = *p.rot_scaling, inv_s2 = 1.0 / (scal * scal);
    for (int i = tid; i < N; i += LT) {
        const double dm = 1.0 - fm[i], lm = rm[i] * dm;
        s_lm += lm;
        double g[3], q[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) { g[c] = p.gt_rot[3 * i + c]; q[c] = p.rs[3 * i + c] * dm; }
        if (p.separate) {
            const double ga = sqrt(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]), qa = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
            double ax = 0;
#pragma unroll
            for (int c = 0; c < 3; ++c) { const double d = g[c] / (ga + 1e-6) - q[c] / (qa + 1e-6); ax += d * d; }
            s_axis += ax * lm;
            s_rot += (ga - qa) * (ga - qa) * lm * inv_s2;
        } else {
#pragma unroll
            for (int c = 0; c < 3; ++c) s_rot += (g[c] - q[c]) * (g[c] - q[c]) * lm * inv_s2;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) { const double d = p.x0[3 * i + c] - p.x[3 * i + c]; s_trans += d * d; }
        for (int a = 0; a < 7; ++a) {
            const double ux = p.ang[(i * 7 + a) * 2], uy = p.ang[(i * 7 + a) * 2 + 1];
            const double n = sqrt(ux * ux + uy * uy), vx = ux / (n + 1e-8), vy = uy / (n + 1e-8);
            const double gx = p.a_gt[(i * 7 + a) * 2], gy = p.a_gt[(i * 7 + a) * 2 + 1];
            const double hx = p.a_alt[(i * 7 + a) * 2], hy = p.a_alt[(i * 7 + a) * 2 + 1];
            const double d1 = (vx - gx) * (vx - gx) + (vy - gy) * (vy - gy), d2 = (vx - hx) * (vx - hx) + (vy - hy) * (vy - hy);
            const double mk = p.a_mask[i * 7 + a];
            s_tor += fmin(d1, d2) * mk;
            s_tm += mk;
        }
    }
    for (int f = tid; f < p.nf; f += LT) {                 // frames with any unmasked residue (:1222 batch_loss_mask)
        bool any = false;
        for (int i = 0; i < N; ++i) any = any || (p.res_mask[(long)f * N + i] != 0.0);
        s_cnt += any ? 1.0 : 0.0;
    }
    s_lm = block_sum(s_lm, red); s_rot = block_sum(s_rot, red); s_axis = block_sum(s_axis, red);
    s_trans = block_sum(s_trans, red); s_tor = block_sum(s_tor, red); s_tm = block_sum(s_tm, red); s_cnt = block_sum(s_cnt, red);

    const double denom = s_lm + 1e-10;
    const double t_gate = (*p.t > p.t_thr) ? 1.0 : 0.0;
    const double k_rot = p.w_rot * t_gate * (double)p.rot_on / denom;      // weight of the (angle | full) rotation term
    const double k_axis = (double)p.rot_on / denom;
    double rot = s_rot * k_rot + (p.separate ? s_axis * k_axis : 0.0);
    double trans = s_trans / (3.0 * N) * p.w_trans;
    const double tor_den = s_tm + 1e-2;
    double tor = s_tor / tor_den * p.w_tor;
    const double g1 = (trans < 100.0) ? 1.0 : 0.0;
    rot *= g1;
    trans *= g1;
    const double g2 = (trans < 100.0) ? 1.0 : 0.0;
    tor *= g2;
    const double fin = rot + trans + tor;
    // the per-frame value is repeated nf times, then summed / (count + 1e-10); the count is an integer tensor, so torch
    // forms that denominator in fp32: exactly the count when it is >= 1, fp32(1e-10) when every frame is empty
    const double nrm = (double)p.nf / (double)((float)s_cnt + 1e-10f);
    if (tid == 0) {
        p.out[0] = fin * nrm; p.out[1] = rot * nrm; p.out[2] = trans * nrm; p.out[3] = tor * nrm;
        p.out[4] = rot; p.out[5] = trans; p.out[6] = tor; p.out[7] = fin;
    }
    // ---- gradients of out[0] ----
    for (int i = tid; i < N; i += LT) {
        const double dm = 1.0 - fm[i], lm = rm[i] * dm;
        double g[3], q[3], dq[3] = {0, 0, 0};
#pragma unroll
        for (int c = 0; c < 3; ++c) { g[c] = p.gt_rot[3 * i + c]; q[c] = p.rs[3 * i + c] * dm; }
        if (p.separate) {
            const double ga = sqrt(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]), qa = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
            // angle term: d (ga - qa)^2 = -2 (ga - qa) q / qa;  axis term: a = q / (qa + e).  At q = 0 the norm's gradient
            // is 0 (torch's convention), which drops the angle term but leaves the axis term's direct part d a / 1e-6.
            double dax[3], dot = 0;
#pragma unroll
            for (int c = 0; c < 3; ++c) { dax[c] = -2.0 * (g[c] / (ga + 1e-6) - q[c] / (qa + 1e-6)); dot += dax[c] * q[c]; }
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                dq[c] = (qa > 0) ? -2.0 * (ga - qa) * q[c] / qa * lm * inv_s2 * k_rot
                                       + (dax[c] / (qa + 1e-6) - q[c] * dot / (qa * (qa + 1e-6) * (qa + 1e-6))) * lm * k_axis
                                 : dax[c] / 1e-6 * lm * k_axis;
            }
        } else {
#pragma unroll
            for (int c = 0; c < 3; ++c) dq[c] = -2.0 * (g[c] - q[c]) * lm * inv_s2 * k_rot;
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            p.d_rs[3 * i + c] = dq[c] * dm * g1 * nrm;
            p.d_x[3 * i + c] = -2.0 * (p.x0[3 * i + c] - p.x[3 * i + c]) / (3.0 * N) * p.w_trans * g1 * nrm;
        }
        for (int a = 0; a < 7; ++a) {
            const double ux = p.ang[(i * 7 + a) * 2], uy = p.ang[(i * 7 + a) * 2 + 1];
            const double n = sqrt(ux * ux + uy * uy), ne = n + 1e-8, vx = ux / ne, vy = uy / ne;
            const double gx = p.a_gt[(i * 7 + a) * 2], gy = p.a_gt[(i * 7 + a) * 2 + 1];
            const double hx = p.a_alt[(i * 7 + a) * 2], hy = p.a_alt[(i * 7 + a) * 2 + 1];
            const double d1 = (vx - gx) * (vx - gx) + (vy - gy) * (vy - gy), d2 = (vx - hx) * (vx - hx) + (vy - hy) * (vy - hy);
            // d min(d1, d2) / d v; a tie splits the gradient evenly between both targets, as torch.minimum does
            const double wx = d1 < d2 ? 2.0 * (vx - gx) : (d1 > d2 ? 2.0 * (vx - hx) : (vx - gx) + (vx - hx));
            const double wy = d1 < d2 ? 2.0 * (vy - gy) : (d1 > d2 ? 2.0 * (vy - hy) : (vy - gy) + (vy - hy));
            const double k = p.a_mask[i * 7 + a] / tor_den * p.w_tor * g2 * nrm;
            // v = u / (n + 1e-8): at u = 0 the norm's gradient is 0 (torch's convention) and only the direct term w / 1e-8 remains
            double dx = wx / ne, dy = wy / ne;
            if (n > 0) {
                const double dot = wx * ux + wy * uy;
                dx = wx / ne - ux * dot / (n * ne * ne);
                dy = wy / ne - uy * dot / (n * ne * ne);
            }
            p.d_ang[(i * 7 + a) * 2] = dx * k;
            p.d_ang[(i * 7 + a) * 2 + 1] = dy * k;
        }
    }
}

}  // namespace
}  // namespace dfold

using namespace dfold;

// All tensors fp64, contiguous; per-residue inputs are those of the LAST frame, the masks cover all nf frames.
// out[8] = {loss, rot, trans, torsion (normalised as the reference's aux_data), rot, trans, torsion, final (per-frame values)};
// d_ang / d_rs / d_x = d out[0] / d (angles, rot_score, translation) of the last frame.
extern "C" int dfold_loss_fwd(const double* ang, const double* a_gt, const double* a_alt, const double* a_mask, const double* rs,
                              const double* gt_rot, const double* x, const double* x0, const double* res_mask,
                              const double* fixed_mask, const double* t, const double* rot_scaling, int nf, int N, double w_tor,
                              double w_rot, double w_trans, double t_thr, int rot_on, int separate, double* out, double* d_ang,
                              double* d_rs, double* d_x, void* stream) {
    DFOLD_REQUIRE(nf > 0 && N > 0, "dfold_loss_fwd: empty problem");
    LossParams p;
    p.ang = ang; p.a_gt = a_gt; p.a_alt = a_alt; p.a_mask = a_mask; p.rs = rs; p.gt_rot = gt_rot; p.x = x; p.x0 = x0;
    p.res_mask = res_mask; p.fixed_mask = fixed_mask; p.t = t; p.rot_scaling = rot_scaling; p.nf = nf; p.N = N;
    p.w_tor = w_tor; p.w_rot = w_rot; p.w_trans = w_trans; p.t_thr = t_thr; p.rot_on = rot_on; p.separate = separate;
    p.out = out; p.d_ang = d_ang; p.d_rs = d_rs; p.d_x = d_x;
    loss_kernel<<<1, LT, 0, as_stream(stream)>>>(p);
    return check_launch("loss_kernel");
}
