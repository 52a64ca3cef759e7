// The advance step of the trajectory rollout (Experiment.eval_extension, train_DFOLD_dynamics.py:931-1000), one launch:
//
//   rollout_advance_kernel   s = *step; if 0 <= s < L:
//                              rigid_traj[s] = rigid_pred[nf - 1]                  (:994, rigid_pred[-1:])
//                              atom_traj[s]  = atom37[nf - 1]                      (:993, atom_pred[-1:])
//                              rigids_0[f]   = rigid_pred[min(f + 1, nf - 1)]      (:996, cat(rigid_pred[1:], rigid_pred[-1:]))
//                              *step = s + 1
//                            otherwise nothing is written.
//
// The row index lives on the device, so one captured CUDA graph (network forward + this launch) serves every step of a
// rollout.  The kernel runs as ONE CTA: every thread reads the counter before thread 0 advances it, with no inter-CTA
// ordering to arrange.  The copies are a few hundred kB at most (2 x 1024 residues: 57 kB of rigids, 454 kB of atoms).
#include <stdint.h>

#include "common.cuh"

namespace dfold {
namespace {

constexpr int kThreads = 1024;

__global__ void __launch_bounds__(kThreads)
rollout_advance_kernel(const float* __restrict__ rigid_pred, const float* __restrict__ atom37, float* __restrict__ rigids_0,
                       float* __restrict__ rigid_traj, float* __restrict__ atom_traj, long long* __restrict__ step, int nf, int N,
                       int A, int L) {
    __shared__ long long s_step;
    if (threadIdx.x == 0) s_step = *step;
    __syncthreads();
    const long long s = s_step;
    if (s < 0 || s >= L) return;                         // uniform over the CTA
    const long fr = 7L * N;                              // floats per frame of rigids
    const long fa = 3L * A * N;                          // floats per frame of atoms
    const long n0 = (long)nf * fr;
    for (long i = threadIdx.x; i < n0; i += kThreads)
        rigids_0[i] = rigid_pred[i < n0 - fr ? i + fr : i];
    const float* last_r = rigid_pred + (long)(nf - 1) * fr;
    float* row_r = rigid_traj + s * fr;
    for (long i = threadIdx.x; i < fr; i += kThreads) row_r[i] = last_r[i];
    const float* last_a = atom37 + (long)(nf - 1) * fa;
    float* row_a = atom_traj + s * fa;
    for (long i = threadIdx.x; i < fa; i += kThreads) row_a[i] = last_a[i];
    __syncthreads();
    if (threadIdx.x == 0) *step = s + 1;
}

}  // namespace
}  // namespace dfold

using namespace dfold;

extern "C" int dfold_rollout_advance(const float* rigid_pred, const float* atom37, float* rigids_0, float* rigid_traj,
                                     float* atom_traj, long long* step, int nf, int N, int A, int L, void* stream) {
    DFOLD_REQUIRE(rigid_pred && atom37 && rigids_0 && rigid_traj && atom_traj && step, "dfold_rollout_advance: null pointer");
    DFOLD_REQUIRE(nf >= 2, "dfold_rollout_advance: need nf >= 2 frames (got %d)", nf);
    DFOLD_REQUIRE(N >= 1 && A >= 1 && L >= 1, "dfold_rollout_advance: need N >= 1, A >= 1 and L >= 1 (got %d, %d, %d)", N, A, L);
    const uintptr_t p = reinterpret_cast<uintptr_t>(rigid_pred), r = reinterpret_cast<uintptr_t>(rigids_0);
    const uintptr_t bytes = (uintptr_t)nf * (uintptr_t)N * 7u * sizeof(float);
    DFOLD_REQUIRE(p + bytes <= r || r + bytes <= p, "dfold_rollout_advance: rigid_pred aliases rigids_0 (the shift is in place)");
    rollout_advance_kernel<<<1, kThreads, 0, as_stream(stream)>>>(rigid_pred, atom37, rigids_0, rigid_traj, atom_traj, step, nf,
                                                                 N, A, L);
    return check_launch("rollout_advance_kernel");
}
