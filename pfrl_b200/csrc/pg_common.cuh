// pg_common.cuh -- one row of a policy-gradient loss's backward, shared by reinforce.cu and
// a3c.cu: given the fp32 gradients c_lp and c_h that the loss hands log pi(a) and H of the
// row, write d loss / d(distribution parameters) of that row.
//   Categorical, z = Categorical._param (normalised logits), p = softmax(z):
//     d log pi(a) / dz = e_a (log_prob is a gather of z)
//     H = -sum_j c_j p_j with c_j = max(z_j, finfo(fp32).min) (torch's clamp), so
//     dH / dz_j = -p_j (m_j + c_j + H), m_j = [z_j >= finfo.min] (the clamp passes the gradient)
//   Independent(Normal(loc, scale), 1), d = a - loc:
//     d log pi / d loc = d / scale^2,  d log pi / d scale = d^2 / scale^3 - 1 / scale
//     dH / d scale = 1 / scale,        dH / d loc = 0
// fp64 arithmetic, fp32 storage.  One warp per row, lanes striding the K categories or the A
// action dimensions.
#pragma once
#include <float.h>
#include <math.h>
#include <stdint.h>

namespace {

constexpr double kHalfLog2Pi = 0.91893853320467274178; // log(sqrt(2 pi))

__device__ __forceinline__ double warp_sum(double v)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ double warp_max(double v)
{
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

struct RowTerms {
    double lp, h; // log pi(a) and H of the row
};

// Row i of a Categorical: args.z [N, K] with K = args.D, int64 args.act [N]; writes args.g_z
// (an action outside [0, K) gives NaN).  H is returned in every lane, log pi(a) (NaN for an
// invalid action) in lane 0.
template <class Args>
__device__ __forceinline__ RowTerms categorical_row_grad(const Args &a, int64_t i, int lane,
                                                         double c_lp, double c_h)
{
    const int K = a.D;
    const size_t row = (size_t)i * K;
    const float *z = a.z + row;
    // softmax statistics of the row: lse of z (0 up to rounding, z being normalised)
    double m = -INFINITY;
    for (int k = lane; k < K; k += 32) m = fmax(m, (double)z[k]);
    m = warp_max(m);
    double s = 0.0;
    for (int k = lane; k < K; k += 32) s += exp((double)z[k] - m);
    const double lse = m + log(warp_sum(s));
    // H = -sum p_j clamp(z_j)
    double h = 0.0;
    for (int k = lane; k < K; k += 32) {
        const double p = exp((double)z[k] - lse);
        h -= p * fmax((double)z[k], (double)-FLT_MAX);
    }
    h = warp_sum(h);
    const int64_t act = a.act[i];
    const bool valid = act >= 0 && act < K;
    for (int k = lane; k < K; k += 32) {
        const double zk = (double)z[k], p = exp(zk - lse);
        const double dh = -p * ((zk >= (double)-FLT_MAX ? 1.0 : 0.0) + fmax(zk, (double)-FLT_MAX) + h);
        double g = c_h * dh;
        if (k == act) g += c_lp;
        a.g_z[row + k] = valid ? (float)g : NAN;
    }
    double lp = 0.0;
    if (lane == 0) lp = valid ? (double)z[act] : NAN;
    return {lp, h};
}

// Row i of an Independent(Normal, 1): args.loc, args.scale (null = 1) and the sampled
// args.act_val [N, A] with A = args.D; writes args.g_loc and, unless null, args.g_scale.
// With want_sums, log pi(a) and H are summed over the row in every lane; otherwise both are
// lane partials.
template <class Args>
__device__ __forceinline__ RowTerms gaussian_row_grad(const Args &a, int64_t i, int lane,
                                                      double c_lp, double c_h, bool want_sums)
{
    const int A = a.D;
    const size_t row = (size_t)i * A;
    double lp = 0.0, h = 0.0;
    for (int k = lane; k < A; k += 32) {
        const double s = a.scale ? (double)a.scale[row + k] : 1.0;
        const double d = (double)a.act_val[row + k] - (double)a.loc[row + k];
        const double inv_s = 1.0 / s, ls = log(s);
        a.g_loc[row + k] = (float)(c_lp * d * inv_s * inv_s);
        if (a.g_scale)
            a.g_scale[row + k] = (float)(c_lp * (d * d * inv_s * inv_s * inv_s - inv_s) + c_h * inv_s);
        lp += -(d * d) * 0.5 * inv_s * inv_s - ls - kHalfLog2Pi;
        h += 0.5 + kHalfLog2Pi + ls;
    }
    if (want_sums) {
        lp = warp_sum(lp);
        h = warp_sum(h);
    }
    return {lp, h};
}

} // namespace
