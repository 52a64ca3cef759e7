// Forward SE(3) diffusion of a training window on the device (the data loader's noising step).
//
//   igso3_tables_kernel      IGSO(3) inverse-cdf tables: cdf [num_sigma][num_omega] and score_scaling [num_sigma], fp64,
//                            one CTA per sigma row.  Replaces src/data/so3_diffuser.py:132-180.
//   forward_marginal_kernel  rigids_0 + time t + draws  ->  rigids_t, rotation / translation scores and their scalings,
//                            one warp per (frame, residue).  Replaces src/data/se3_diffuser.py:47-110 (forward_marginal)
//                            and :217-280 (sample_ref), so3_diffuser.py:215-251, :274-327, r3_diffuser.py:39-40, :81-104,
//                            :159-177, and the scipy rotation-vector round trips of se3_diffuser.py:11-29 / utils.py:184-195.
//
// The random draws are inputs (axis normals, uniforms, translation normals, all fp64), so the launch is graph-capturable
// and a caller can reproduce the reference's numpy stream exactly by injecting it.
#include "common.cuh"
#include "igso3.cuh"

namespace dfold {
namespace {

constexpr double kPi = 3.141592653589793;

// ------------------------------------------------------------------------------------------------------------
// IGSO(3) tables.  Row i (sigma = discrete_sigma[i]), angle j: omega_j = (j + 1) pi / num_omega (np.linspace(0, pi,
// num_omega + 1)[1:], whose last point is pi exactly);
//   E_j  = sum_l (2l+1) exp(-l(l+1) sigma^2/2) sin(omega_j (l+1/2)) / sin(omega_j/2)        (igso3_expansion)
//   dE_j = the same series differentiated in omega                                             (score)
//   pdf_j = E_j (1 - cos omega_j) / pi,   sn_j = dE_j / (E_j + 1e-4)
//   cdf_j = (pdf_0 + ... + pdf_j) / num_omega * pi
//   score_scaling = sqrt(|sum_j sn_j^2 pdf_j / sum_j pdf_j|) / sqrt(3)
// Summation order (fixed, so equal inputs give equal bits): E_j and dE_j by one thread each, l ascending; the prefix sum
// and both row sums by thread 0, j ascending.  The weights (2l+1) exp(..) depend on (sigma, l) only: staged once per row.
// ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) igso3_tables_kernel(const double* __restrict__ sigma_grid, int num_omega, int L,
                                                           double* __restrict__ cdf, double* __restrict__ score_scaling) {
    extern __shared__ double smem[];
    double* s_decay = smem;                    // [L]
    double* s_pdf = s_decay + L;               // [num_omega]
    double* s_w = s_pdf + num_omega;           // [num_omega]  sn^2 pdf
    __shared__ int s_lc;
    const int row = blockIdx.x;
    const double sigma = sigma_grid[row];
    const double s2h = sigma * sigma * 0.5;
    if (threadIdx.x == 0) s_lc = L;
    __syncthreads();
    for (int l = threadIdx.x; l < L; l += blockDim.x) {
        const double ex = igso3_exponent(l, s2h);
        s_decay[l] = ex < kIgso3ExpCut ? 0.0 : igso3_decay(l, ex);
        if (ex < kIgso3ExpCut) atomicMin(&s_lc, l);          // first vanishing term (the exponent decreases with l)
    }
    __syncthreads();
    const int lc = s_lc;
    const double step = kPi / (double)num_omega;
    for (int j = threadIdx.x; j < num_omega; j += blockDim.x) {
        const double omega = j == num_omega - 1 ? kPi : (double)(j + 1) * step;
        const Igso3Angle<double> a = igso3_angle(omega);
        double e = 0.0, de = 0.0, unused = 0.0;
        for (int l = 0; l < lc; ++l) igso3_term<double, false>(a, l, s_decay[l], e, de, unused);
        const double pdf = e * (1.0 - cos(omega)) / kPi;
        const double sn = de / (e + 1e-4);
        s_pdf[j] = pdf;
        s_w[j] = __dmul_rn(__dmul_rn(sn, sn), pdf);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double acc = 0.0, wsum = 0.0;
        double* out = cdf + (long)row * num_omega;
        for (int j = 0; j < num_omega; ++j) {
            acc += s_pdf[j];
            wsum += s_w[j];
            out[j] = acc / (double)num_omega * kPi;
        }
        score_scaling[row] = sqrt(fabs(wsum / acc)) / sqrt(3.0);
    }
}

// ------------------------------------------------------------------------------------------------------------
// forward marginal
// ------------------------------------------------------------------------------------------------------------
struct FwdParams {
    const float* rigids_0;       // [n,7] (w,x,y,z, tx,ty,tz); NULL in sample_ref mode
    const double* z_axis;        // [n,3] standard normals of the rotation axis (so3 randn(n,3))
    const double* u;             // [n]   uniforms in [0,1) of the angle (so3 rand(n))
    const double* z_trans;       // [n,3] standard normals of the translation (r3 normal(size=(n,3)))
    const float* mask;           // [n] diffuse mask or NULL
    const double* t;             // device scalar
    const double* grid;          // [G] discrete_sigma
    const double* cdf;           // [G][num_omega]
    const double* score_scaling; // [G]
    int G, num_omega, L;
    double e_max, e_min;         // exp(max_sigma), exp(min_sigma)
    double min_b, max_b;         // VP-SDE schedule
    float r3_scale;              // coordinate_scaling
    int diffuse_rot, diffuse_trans, ref_mode;
    float* rigids_t;             // [n,7]
    double* rot_score;           // [n,3]  (NULL allowed in sample_ref mode)
    double* trans_score;         // [n,3]
    double* rot_scaling;         // device scalar
    double* trans_scaling;       // device scalar
    long n;
};

// np.interp(u, xp, fp) with fp[j] = omega_j (compiled_base.c arr_interp): j = last index with xp[j] <= u;
// u < xp[0] -> fp[0]; u > xp[-1] -> fp[-1]; j == len-1 or xp[j] == u -> fp[j];
// else slope = (fp[j+1] - fp[j]) / (xp[j+1] - xp[j]), slope (u - xp[j]) + fp[j] (then the NaN fall-backs).
__device__ __forceinline__ double interp_omega(double u, const double* xp, int len) {
    const double step = kPi / (double)len;
    auto fp = [&](int j) { return j == len - 1 ? kPi : (double)(j + 1) * step; };
    if (u > xp[len - 1]) return kPi;
    if (u < xp[0]) return fp(0);
    int lo = 0, hi = len;
    while (lo < hi) {
        const int mid = lo + ((hi - lo) >> 1);
        if (u >= xp[mid]) lo = mid + 1; else hi = mid;
    }
    const int j = lo - 1;
    if (j == len - 1) return fp(j);
    if (xp[j] == u) return fp(j);
    const double slope = __ddiv_rn(__dsub_rn(fp(j + 1), fp(j)), __dsub_rn(xp[j + 1], xp[j]));
    double r = __dadd_rn(__dmul_rn(slope, __dsub_rn(u, xp[j])), fp(j));
    if (isnan(r)) {
        r = __dadd_rn(__dmul_rn(slope, __dsub_rn(u, xp[j + 1])), fp(j + 1));
        if (isnan(r) && fp(j) == fp(j + 1)) r = fp(j);
    }
    return r;
}

__global__ void __launch_bounds__(256) forward_marginal_kernel(const FwdParams p) {
    extern __shared__ double s_cdf[];          // the cdf row of sigma(t), shared by the CTA's 8 warps
    const double t = *p.t;
    const int sidx = sigma_index(t, p.grid, p.G, p.e_max, p.e_min);
    if (p.diffuse_rot) {
        const double* row = p.cdf + (long)sidx * p.num_omega;
        for (int j = threadIdx.x; j < p.num_omega; j += blockDim.x) s_cdf[j] = row[j];
        __syncthreads();
    }
    // beta(t) = t min_b + t^2 (max_b - min_b) / 2 and the Gaussian marginal's factors (r3_diffuser.py:42-43, :159-167)
    const double beta = __dadd_rn(__dmul_rn(t, p.min_b), __dmul_rn(__dmul_rn(0.5, __dmul_rn(t, t)), p.max_b - p.min_b));
    const double decay = exp(-0.5 * beta);
    const double var = 1.0 - exp(-beta);
    if (blockIdx.x == 0 && threadIdx.x == 0 && !p.ref_mode) {
        *p.rot_scaling = p.diffuse_rot ? p.score_scaling[sidx] : 1.0;
        *p.trans_scaling = p.diffuse_trans ? 1.0 / sqrt(var) : 1.0;
    }
    const long i = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= p.n) return;
    const int lane = threadIdx.x & 31;
    const float m = p.mask ? p.mask[i] : 1.f;
    const double md = (double)m;

    // ---- rotation: v = axis * omega, axis = z / |z| (fp64), omega = np.interp(u, cdf[sigma_idx], discrete_omega) ----
    double q0w = 1.0, q0x = 0.0, q0y = 0.0, q0z = 0.0;
    if (!p.ref_mode) {
        const float* r0 = p.rigids_0 + 7 * i;
        q0w = r0[0]; q0x = r0[1]; q0y = r0[2]; q0z = r0[3];
    }
    double qw = q0w, qx = q0x, qy = q0y, qz = q0z;
    if (p.diffuse_rot) {
        const double zx = p.z_axis[3 * i], zy = p.z_axis[3 * i + 1], zz = p.z_axis[3 * i + 2];
        const double nz = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(zx, zx), __dmul_rn(zy, zy)), __dmul_rn(zz, zz)));
        const double ax = zx / nz, ay = zy / nz, az = zz / nz;
        const double ang = interp_omega(p.u[i], s_cdf, p.num_omega);
        const double vx = ax * ang, vy = ay * ang, vz = az * ang;
        if (p.rot_score) {
            // torch_score in fp64 (so3_diffuser.py:292,303-305): omega = |v| + 1e-6, score = dlog(IGSO3)/domega * v / (omega + 1e-6)
            const double omega = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(vx, vx), __dmul_rn(vy, vy)), __dmul_rn(vz, vz))) + 1e-6;
            double S, dS, d2S;
            igso3_series<double, false>(omega, p.grid[sidx], p.L, lane, S, dS, d2S);
            if (lane < 3) {
                const double g = dS / (S + 1e-4);
                const double v = lane == 0 ? vx : (lane == 1 ? vy : vz);
                p.rot_score[3 * i + lane] = g * v / (omega + 1e-6) * md;
            }
        }
        // R_t = R_0 Exp(v) (right multiplication, so3_diffuser.py:325-326): q_t = q_0 (x) (cos(omega/2), sin(omega/2) axis)
        const double n0 = sqrt(q0w * q0w + q0x * q0x + q0y * q0y + q0z * q0z);
        const double aw = q0w / n0, axq = q0x / n0, ayq = q0y / n0, azq = q0z / n0;
        double sh, ch;
        sincos(0.5 * ang, &sh, &ch);
        const double pw = ch, px = sh * ax, py = sh * ay, pz = sh * az;
        qw = aw * pw - axq * px - ayq * py - azq * pz;
        qx = aw * px + axq * pw + ayq * pz - azq * py;
        qy = aw * py - axq * pz + ayq * pw + azq * px;
        qz = aw * pz + axq * py - ayq * px + azq * pw;
        const double nn = sqrt(qw * qw + qx * qx + qy * qy + qz * qz);
        const double sg = qw < 0.0 ? -1.0 : 1.0;                   // w >= 0 (the reference's eigh leaves the sign arbitrary)
        qw = sg * qw / nn; qx = sg * qx / nn; qy = sg * qy / nn; qz = sg * qz / nn;
    } else if (p.rot_score && lane < 3) {
        p.rot_score[3 * i + lane] = 0.0;
    }

    // ---- translation: x_t = N(e^{-beta/2} s x_0, 1 - e^{-beta}) in scaled units, returned unscaled ----
    if (lane < 3) {
        const float x0f = p.ref_mode ? 0.f : p.rigids_0[7 * i + 4 + lane];
        double xt = (double)x0f;
        if (p.diffuse_trans) {
            const double z = p.z_trans[3 * i + lane];
            if (p.ref_mode) {
                xt = z / (double)p.r3_scale;                                     // sample_ref: randn / coordinate_scaling
            } else {
                const double xs = (double)__fmul_rn(x0f, p.r3_scale);            // fp32 x_0 * scaling, as numpy computes it
                const double xts = __dadd_rn(__dmul_rn(decay, xs), __dmul_rn(sqrt(var), z));   // loc + scale * gauss
                if (p.trans_score) p.trans_score[3 * i + lane] = -__dsub_rn(xts, __dmul_rn(decay, xs)) / var * md;
                xt = xts / (double)p.r3_scale;
                // _apply_mask: m x_t + (1 - m) x_0 (se3_diffuser.py:88-91, 126-127)
                xt = __dadd_rn(__dmul_rn(md, xt), __dmul_rn(1.0 - md, (double)x0f));
            }
        } else if (p.trans_score) {
            p.trans_score[3 * i + lane] = 0.0;
        }
        p.rigids_t[7 * i + 4 + lane] = (float)xt;
    }
    // rotations of residues with mask 0 keep rigids_0 bit for bit (the reference's rotation-vector blend, se3_diffuser.py:
    // 86-87, reduces to selection for a 0/1 mask)
    if (lane == 0) {
        float* o = p.rigids_t + 7 * i;
        if (p.diffuse_rot && (p.ref_mode || m > 0.5f)) {
            o[0] = (float)qw; o[1] = (float)qx; o[2] = (float)qy; o[3] = (float)qz;
        } else {
            o[0] = (float)q0w; o[1] = (float)q0x; o[2] = (float)q0y; o[3] = (float)q0z;
        }
    }
}

}  // namespace
}  // namespace dfold

using namespace dfold;

extern "C" int dfold_igso3_tables(const double* sigma_grid, int num_sigma, int num_omega, int L, double* cdf, double* score_scaling,
                                  void* stream) {
    DFOLD_REQUIRE(sigma_grid && cdf && score_scaling, "dfold_igso3_tables: null pointer");
    DFOLD_REQUIRE(num_sigma > 0 && num_omega > 1 && L > 0, "dfold_igso3_tables: need num_sigma >= 1, num_omega >= 2, L >= 1");
    const size_t smem = ((size_t)L + 2 * (size_t)num_omega) * sizeof(double);
    DFOLD_REQUIRE(smem <= 227 * 1024, "dfold_igso3_tables: L + 2 num_omega = %zu doubles exceed the 227 KB of shared memory",
                  smem / sizeof(double));
    static SmemCfg cfg;
    if (ensure_dyn_smem(igso3_tables_kernel, smem, cfg, "igso3_tables_kernel")) return 1;
    igso3_tables_kernel<<<(unsigned)num_sigma, 256, smem, as_stream(stream)>>>(sigma_grid, num_omega, L, cdf, score_scaling);
    return check_launch("igso3_tables_kernel");
}

extern "C" int dfold_forward_marginal(const float* rigids_0, const double* z_axis, const double* u, const double* z_trans,
                                      const float* mask, const double* t, const double* sigma_grid, const double* cdf,
                                      const double* score_scaling, int num_sigma, int num_omega, int L, double max_sigma,
                                      double min_sigma, double min_b, double max_b, float r3_scale, int diffuse_rot,
                                      int diffuse_trans, int ref_mode, float* rigids_t, double* rot_score, double* trans_score,
                                      double* rot_scaling, double* trans_scaling, long n, void* stream) {
    DFOLD_REQUIRE(n > 0 && num_sigma > 0 && num_omega > 1 && L > 0, "dfold_forward_marginal: empty problem");
    DFOLD_REQUIRE(t && sigma_grid && rigids_t, "dfold_forward_marginal: t / sigma grid / output missing");
    DFOLD_REQUIRE(r3_scale != 0.f, "dfold_forward_marginal: zero coordinate scaling");
    DFOLD_REQUIRE(!diffuse_rot || (cdf && z_axis && u), "dfold_forward_marginal: cdf table / rotation draws missing");
    DFOLD_REQUIRE(!diffuse_trans || z_trans, "dfold_forward_marginal: translation draws missing");
    if (ref_mode) {
        DFOLD_REQUIRE(diffuse_rot && diffuse_trans && mask == nullptr, "dfold_forward_marginal: sample_ref needs both diffusions and no mask");
    } else {
        DFOLD_REQUIRE(rigids_0 && rot_score && trans_score && rot_scaling && trans_scaling && score_scaling,
                      "dfold_forward_marginal: rigids_0 / score outputs missing");
    }
    const size_t smem = diffuse_rot ? (size_t)num_omega * sizeof(double) : 0;
    DFOLD_REQUIRE(smem <= 227 * 1024, "dfold_forward_marginal: num_omega = %d exceeds the shared-memory row", num_omega);
    static SmemCfg cfg;
    if (ensure_dyn_smem(forward_marginal_kernel, smem, cfg, "forward_marginal_kernel")) return 1;
    FwdParams p{rigids_0, z_axis, u, z_trans, mask, t, sigma_grid, cdf, score_scaling, num_sigma, num_omega, L,
                exp(max_sigma), exp(min_sigma), min_b, max_b, r3_scale, diffuse_rot, diffuse_trans, ref_mode,
                rigids_t, ref_mode ? nullptr : rot_score, ref_mode ? nullptr : trans_score, rot_scaling, trans_scaling, n};
    forward_marginal_kernel<<<(unsigned)cdiv(n, 8), 256, smem, as_stream(stream)>>>(p);
    return check_launch("forward_marginal_kernel");
}
