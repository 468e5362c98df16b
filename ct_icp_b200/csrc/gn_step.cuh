// gn_step.cuh — the serial tail of a Gauss-Newton iteration, one warp: normal equations from the accumulator, motion-model
// regularisers, the 12x12 solve, the Euler-ZYX pose update and the stop test (DoRegisterGaussNewton, ct_icp.cpp:860-980).
// Included by icp_gn.cu (k_gn_solve / k_gn_persistent); a header so that the device routine can be tested on its own.
#pragma once
#include "icp.h"
#include "se3.cuh"
#include "small_solve.cuh"

namespace cticp {

__device__ __forceinline__ M3 euler_from_sincos(double sa, double ca, double sb, double cb, double sg, double cg) {
    M3 R;   // ct_icp.cpp:916-932
    R.m[0][0] = cg * cb; R.m[0][1] = -sg * ca + cg * sb * sa; R.m[0][2] = sg * sa + cg * sb * ca;
    R.m[1][0] = sg * cb; R.m[1][1] = cg * ca + sg * sb * sa;  R.m[1][2] = -cg * sa + sg * sb * ca;
    R.m[2][0] = -sb;     R.m[2][1] = cb * sa;                 R.m[2][2] = cb * ca;
    return R;
}

// One warp: accumulator (96 doubles in `acc`) → normal equations → GN step → pose update (ct_icp.cpp:860-980).
// mode 0: full step. mode 1: only emit the linear system into sys_out (debug tap).
__device__ __noinline__ void warp_gn_solve(const double *acc, SolveScratch &S, IcpState *st, const GnParams &P, int mode,
                              double *sys_out, int lane) {
    const int n_used = (int) (acc[kAccUsed] + 0.5);
    if (lane == 0) {
        st->n_used = n_used;
        st->n_keypoints = (int) (acc[kAccKeypoints] + 0.5);
        st->stat_keypoint_iters += (unsigned long long) (acc[kAccKeypoints] + 0.5);
        st->stat_stencil_points += (unsigned long long) (acc[kAccStencil] + 0.5);
        if (sys_out) sys_out[156] = (double) n_used;
    }
    if (n_used < 100) {   // ct_icp.cpp:860-871
        if (lane == 0) {
            st->failed = 1;
            st->done = 1;
        }
        return;
    }
    {
        const double inv = 1.0 / (double) n_used;   // :877-882
        for (int e = lane; e < 78; e += 32) {
            const int i = c_pair_i[e], j = c_pair_j[e];
            const double v = acc[e] * inv;
            S.A[i][j] = v;
            S.A[j][i] = v;
        }
        if (lane < 12) S.b[lane] = acc[78 + lane] * inv;
    }
    __syncwarp();
    if (st->has_motion_model && lane < 3) {   // :885-910
        const int d = lane;
        const double ac = st->beta_location, ae = st->beta_cv;
        const double diff_traj = st->tb[d] - st->te[d];   // the frame's own begin - end (sic, :892)
        S.A[3 + d][3 + d] += ac;
        S.b[3 + d] -= ac * diff_traj;
        const double diff_ego = st->te[d] - st->tb[d] - st->prev_te[d] + st->prev_tb[d];
        S.A[9 + d][9 + d] += ae;
        S.b[9 + d] -= ae * diff_ego;
    }
    __syncwarp();
    if (sys_out) {
        for (int e = lane; e < 144; e += 32) sys_out[e] = S.A[e / 12][e % 12];
        if (lane < 12) sys_out[144 + lane] = S.b[lane];
    }
    if (mode == 1) return;

    CT_STAMP(const long long t_ldlt = clock64();)
    warp_ldlt_solve12(S, lane);   // :914
    CT_STAMP(if (lane == 0) st->dbg_t[2] += (unsigned long long) (clock64() - t_ldlt);)
    CT_STAMP(const long long t_pose = clock64();)
    {
        // A rank-deficient system (all keypoints on one plane and no regulariser, …) gives a non-finite step where Eigen's
        // pivoted LDL^T would still return something bounded: report the failure instead of propagating NaN poses
        const bool finite = lane >= 12 || isfinite(S.x[lane]);
        if (!__all_sync(0xffffffffu, finite)) {
            if (lane == 0) {
                st->failed = 4;
                st->done = 1;
            }
            return;
        }
    }

    if (lane < 6) {   // angles x[0..2] (begin) and x[6..8] (end): sin / cos evaluated by six lanes at once
        const double ang = S.x[lane < 3 ? lane : lane + 3];
        // a GN step's angles are a fraction of a degree: polynomials (se3.cuh) instead of libm's argument reduction
        const bool small = fabs(ang) <= 0.5;
        S.sn[lane] = small ? sin_upto_half(ang) : sin(ang);
        S.cs[lane] = small ? cos_upto_half(ang) : cos(ang);
    }
    __syncwarp();
    if (lane < 2) {   // lane 0: begin pose, lane 1: end pose (:916-962)
        const int o = 3 * lane;
        const M3 R = euler_from_sincos(S.sn[o], S.cs[o], S.sn[o + 1], S.cs[o + 1], S.sn[o + 2], S.cs[o + 2]);
        double *qp = lane == 0 ? st->qb : st->qe;
        double *tp = lane == 0 ? st->tb : st->te;
        const Q4 q = qnormalized(qfromR(mmul(R, qtoR(Q4{qp[0], qp[1], qp[2], qp[3]}))));
        qp[0] = q.x; qp[1] = q.y; qp[2] = q.z; qp[3] = q.w;
        const int xo = lane == 0 ? 3 : 9;
        for (int d = 0; d < 3; ++d) tp[d] += S.x[xo + d];
    }
    __syncwarp();
    if (lane == 0) {
        double nrm = 0;
        for (int i = 0; i < 12; ++i) nrm += S.x[i] * S.x[i];
        nrm = sqrt(nrm);
        st->x_norm = nrm;
        st->iter += 1;
        if (nrm < P.threshold_norm) st->done = 1;   // :978
        const SlerpConsts sc = slerp_consts(Q4{st->qb[0], st->qb[1], st->qb[2], st->qb[3]},
                                            Q4{st->qe[0], st->qe[1], st->qe[2], st->qe[3]});
        st->slerp_theta = sc.theta;
        st->slerp_inv_sin = sc.inv_sin;
        st->slerp_linear = sc.linear;
        st->slerp_negate = sc.negate;
        CT_STAMP(st->dbg_t[3] += (unsigned long long) (clock64() - t_pose);)
    }
}

}  // namespace cticp
