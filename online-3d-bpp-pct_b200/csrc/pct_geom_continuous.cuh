// Continuous-domain geometry policy of the stability routine (pct_stability.cuh), the 6-decimal rounding and the resting-height loops:
// shared by the kernels of pct_continuous.cu and by the host build of the routine that the CPU tests drive (tests/host_emul/).
#pragma once
#include <cstdint>
#include "pct_kernels.h"
#include "pct_stability.cuh"

namespace pct {

// np.around(v, 6) = rint(v * 1e6) / 1e6.  The correctly rounded IEEE division is a ~30-instruction subroutine on the GPU and was a large share of the
// continuous feasibility kernel's warp instructions.  For the constant divisor 1e6 the quotient of an integer-valued a follows
// from the correctly rounded reciprocal y = 1e-6 by one FMA correction (Markstein): q0 = a * y, r = fma(-q0, 1e6, a) (exact), q = fma(r, y, q0).
// scratch/around6_exhaustive.c checks q == a / 1e6 for EVERY integer |a| <= 2.2e9 (|v| <= 2200 at 6 decimals): 0 mismatches (q0 alone: 30 %); beyond
// that range the exact division runs.  tests/test_oracle_units.py::test_fast_around6_equals_the_division samples it through the host build.
__device__ __forceinline__ double around6(double v) {
    const double a = rint(v * 1e6);
    if (fabs(a) <= 2.2e9) {
        const double q0 = a * 1e-6;
        if (a == 0.0) return q0;  // keeps the sign of a zero numerator like the division does
        return fma(fma(-q0, 1e6, a), 1e-6, q0);
    }
    return ddiv(a, 1e6);
}

// ---- geometry policy for the stability routine -------------------------------------------------------------
struct NodeC { double lx, ly, lz, dx, dy, dz, mass; };
struct GeomC {
    typedef NodeC Node;
    const double (*box)[6];
    const double *den;
    int n;
    __device__ __forceinline__ int n_boxes() const { return n; }
    __device__ __forceinline__ void node_box(int id, NodeC &o) const {
        const double *b = box[id];
        o.lx = b[0]; o.ly = b[1]; o.lz = b[2]; o.dx = b[3]; o.dy = b[4]; o.dz = b[5];
        o.mass = b[3] * b[4] * b[5] * den[id];  // C:space.py:34
    }
    __device__ __forceinline__ void centre(const NodeC &o, double &cx, double &cy, double &cz) const {  // C:space.py:31
        cx = o.lx + o.dx * 0.5; cy = o.ly + o.dy * 0.5; cz = o.lz + o.dz * 0.5;
    }
    // interSect2D + the support filter of drop_box (C:space.py:305-314, 350-359)
    __device__ __noinline__ bool support(const NodeC &nd, int t, double r[4]) const {
        const double *b = box[t];
        if (!(fabs(b[2] + b[5] - nd.lz) < 1e-6)) return false;
        const double i0 = around6(fmin(-nd.lx, -b[0])), i1 = around6(fmin(-nd.ly, -b[1]));
        const double i2 = around6(fmin(nd.lx + nd.dx, b[0] + b[3])), i3 = around6(fmin(nd.ly + nd.dy, b[1] + b[4]));
        if (!((i0 + i2 > 0) && (i1 + i3 > 0))) return false;
        r[0] = -i0; r[1] = -i1; r[2] = i2; r[3] = i3;
        return true;
    }
    __device__ __forceinline__ bool strictly_inside(double cx, double cy, const double r[4]) const {  // C:space.py:85-86
        return cx - r[0] > 1e-6 && r[2] - cx > 1e-6 && cy - r[1] > 1e-6 && r[3] - cy > 1e-6;
    }
};

// resting height: max top over the boxes whose rounded footprint intersection is positive (interSect2D)
__device__ __forceinline__ double rest_height_c(const double (*box)[6], int first, int n, int stride, double lx, double ly, double hx, double hy) {
    double mh = 0;
    bool any = false;
    for (int t = first; t < n; t += stride) {
        const double *b = box[t];
        const double i0 = around6(fmin(-lx, -b[0])), i1 = around6(fmin(-ly, -b[1]));
        const double i2 = around6(fmin(hx, b[0] + b[3])), i3 = around6(fmin(hy, b[1] + b[4]));
        if ((i0 + i2 > 0) && (i1 + i3 > 0)) {
            const double top = b[2] + b[5];
            if (!any || top > mh) mh = top;
            any = true;
        }
    }
    return any ? mh : -1.0;  // -1: no overlap (the reference returns 0 then)
}

// The same resting height from PRE-ROUNDED operands.  around6 is monotone non-decreasing (IEEE multiply by 1e6, rint and the
// correctly rounded division by 1e6 all are), and a monotone f commutes with min: f(min(a, b)) == min(f(a), f(b)).  Hence
//   around6(fmin(-lx, -b[0])) == fmin(around6(-lx), around6(-b[0]))        (bit for bit, for every input)
// and the four roundings per (placement, box) pair of interSect2D become four per placement + four per box, the latter
// computed once per launch into shared memory (rb[t] = {around6(-lx_t), around6(-ly_t), around6(hx_t), around6(hy_t), top_t}).
// tests/test_oracle_units.py::test_around6_commutes_with_min checks the identity on the host.
__device__ __forceinline__ double rest_height_pre(const double (*rb)[5], int n, double c0, double c1, double c2, double c3) {
    double mh = 0;
    bool any = false;
    for (int t = 0; t < n; t++) {
        const double *b = rb[t];
        const double i0 = fmin(c0, b[0]), i1 = fmin(c1, b[1]), i2 = fmin(c2, b[2]), i3 = fmin(c3, b[3]);
        if ((i0 + i2 > 0) && (i1 + i3 > 0)) {
            const double top = b[4];
            if (!any || top > mh) mh = top;
            any = true;
        }
    }
    return any ? mh : -1.0;
}

}  // namespace pct
