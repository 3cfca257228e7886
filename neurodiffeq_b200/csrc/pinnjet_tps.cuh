// pinnjet_tps.cuh -- arguments of the field kernel (pinnjet_tps.cu): thin-plate-spline maps of irregular-domain conditions
// and their first and second derivatives at every point, the rows the residual programs read with OP_FIELD.
#pragma once
#include <cuda_runtime.h>
#include "../../include/pinnjet.h"

namespace pj {

template <typename R>
struct TpsGroupK {
    const R* centres;   // [m][2]
    const R* coefs;     // [k][m + 3]
    int m, k, cx, cy;
    R s2;
};

template <typename R>
struct TpsArgs {
    const R* coords[PJ_MAX_COORDS];
    long long n;
    int n_groups, n_rows;
    TpsGroupK<R> group[PJ_MAX_TPS_GROUPS];
    int4 row[PJ_MAX_FIELD_ROWS];   // (group, map, derivative, -): PjFieldRow
    R* out;                        // [n_rows][n]
};

cudaError_t launch_tps_fields(const TpsArgs<float>& a, cudaStream_t s);
cudaError_t launch_tps_fields(const TpsArgs<double>& a, cudaStream_t s);

}  // namespace pj
