// sx_log_sum.cuh -- the reference's double log-sum, restated with its libm (sx_libm_mirror_d.h), bit for bit.  Used by K5 and K5b.
#pragma once

#include "sx_device_util.cuh"

__device__ __forceinline__ double log1p_switch_d(double x) // blt_util/math_util.hh:33-47
{
    return (fabs(x) < 0.01) ? sx_log1p(x) : sx_log(d_add(1.0, x)); // (the reference's libm, bit for bit: sx_libm_mirror_d.h)
}
__device__ __forceinline__ double get_log_sum(double x1, double x2) // blt_util/logSumUtil.hh:33-41
{
    if (x1 < x2)
    {
        const double t = x1;
        x1 = x2;
        x2 = t;
    }
    return d_add(x1, log1p_switch_d(sx_exp(d_sub(x2, x1))));
}
