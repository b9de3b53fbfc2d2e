// Device recurrences: one normalised Taylor derivative ("coefficient") of one u variable at one order,
// for the N adjacent lanes owned by the calling thread. Each opcode is the hand-written counterpart of one
// taylor_c_diff_func_* of the reference (compact-mode, i.e. running-accumulator, summation order):
//
//   sum / sub                       src/math/sum.cpp:250-371, src/detail/sub.cpp:180-398
//   k*v, -v, v*v                    src/math/prod.cpp:443-705
//   div                             src/detail/div.cpp:189-431
//   square / sqrt / pow             src/math/pow.cpp:618-963; order-0 evaluation :292-355, :136-152
//   sum_sq                          src/detail/sum_sq.cpp:250-468
//   sin / cos / tanh / exp / log    src/math/sin.cpp:241-372, cos.cpp:241-372, tanh.cpp:183-318,
//                                   exp.cpp:150-285, log.cpp:164-305
//   time / constant-only functions  src/math/time.cpp:82-104, include/heyoka/detail/taylor_common.hpp:88-157
//
// Floating-point contract: this file is compiled with -fmad=false, so the ONLY fused operations are
// the explicit fma() calls below: every `acc + a*b` of the reference's accumulation loops is
// fma(a, b, acc) (a contraction LLVM is allowed to make in the reference, src/llvm_state.cpp:842-845);
// everything else rounds after each operation. tests/ compare against the oracle's sequential+FMA mode.
//
// Storage is abstracted by a Tape policy (two implementations, see batch.cu):
//   tape.row(ref) -> Row          the coefficients of one u variable for this thread's lanes
//   row.at(o)     -> vd<N>        coefficient of order o          row.set(o, v)
//   tape.par(idx), tape.time()    runtime parameter / time of the lanes
//   tape.arg(i), tape.cst(i)      entries of the program's argument table / constant pool
// `ref` is whatever the program stores in an op's operand fields: a u-variable index for the HBM tape,
// a packed slot reference for the shared-memory tape.
#ifndef HEYOKA_B200_CSRC_RECURRENCES_CUH
#define HEYOKA_B200_CSRC_RECURRENCES_CUH

#include <cstdint>

#include "device_program.cuh"

namespace heyoka_b200::dev
{

// N adjacent lanes' worth of doubles, with element-wise arithmetic.
template <int N>
struct vd {
    double v[N];
};

#define HY_VD_BINOP(op)                                                                                                \
    template <int N>                                                                                                   \
    __device__ __forceinline__ vd<N> operator op(const vd<N> &a, const vd<N> &b)                                       \
    {                                                                                                                  \
        vd<N> r;                                                                                                       \
        _Pragma("unroll") for (int i = 0; i < N; ++i) r.v[i] = a.v[i] op b.v[i];                                       \
        return r;                                                                                                      \
    }                                                                                                                  \
    template <int N>                                                                                                   \
    __device__ __forceinline__ vd<N> operator op(const vd<N> &a, double b)                                             \
    {                                                                                                                  \
        vd<N> r;                                                                                                       \
        _Pragma("unroll") for (int i = 0; i < N; ++i) r.v[i] = a.v[i] op b;                                            \
        return r;                                                                                                      \
    }                                                                                                                  \
    template <int N>                                                                                                   \
    __device__ __forceinline__ vd<N> operator op(double a, const vd<N> &b)                                             \
    {                                                                                                                  \
        vd<N> r;                                                                                                       \
        _Pragma("unroll") for (int i = 0; i < N; ++i) r.v[i] = a op b.v[i];                                            \
        return r;                                                                                                      \
    }

HY_VD_BINOP(+)
HY_VD_BINOP(-)
HY_VD_BINOP(*)
HY_VD_BINOP(/)
#undef HY_VD_BINOP

template <int N>
__device__ __forceinline__ vd<N> operator-(const vd<N> &a)
{
    vd<N> r;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        r.v[i] = -a.v[i];
    }
    return r;
}

template <int N>
__device__ __forceinline__ vd<N> splat(double x)
{
    vd<N> r;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        r.v[i] = x;
    }
    return r;
}

// fma(a, b, c) element-wise; scalar first factor overload for the weighted sums.
template <int N>
__device__ __forceinline__ vd<N> vfma(const vd<N> &a, const vd<N> &b, const vd<N> &c)
{
    vd<N> r;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        r.v[i] = ::fma(a.v[i], b.v[i], c.v[i]);
    }
    return r;
}
template <int N>
__device__ __forceinline__ vd<N> vfma(double a, const vd<N> &b, const vd<N> &c)
{
    vd<N> r;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        r.v[i] = ::fma(a, b.v[i], c.v[i]);
    }
    return r;
}

#define HY_VD_MAP1(name, fn)                                                                                           \
    template <int N>                                                                                                   \
    __device__ __forceinline__ vd<N> name(const vd<N> &a)                                                              \
    {                                                                                                                  \
        vd<N> r;                                                                                                       \
        _Pragma("unroll") for (int i = 0; i < N; ++i) r.v[i] = fn(a.v[i]);                                             \
        return r;                                                                                                      \
    }
HY_VD_MAP1(vsqrt, ::sqrt)
HY_VD_MAP1(vsin, ::sin)
HY_VD_MAP1(vcos, ::cos)
HY_VD_MAP1(vtanh, ::tanh)
HY_VD_MAP1(vexp, ::exp)
HY_VD_MAP1(vlog, ::log)
// sigmoid(x) = 1 / (1 + exp(-x)) (src/math/sigmoid.cpp:69-75).
template <int N>
__device__ __forceinline__ vd<N> vsigmoid(const vd<N> &x)
{
    vd<N> r;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        r.v[i] = 1. / (1. + ::exp(-x.v[i]));
    }
    return r;
}
// (Leaky) ReLU of `val` gated by the sign of `x0` (src/math/relu.cpp:118-128, :157-176): x0 > 0 ? val : slope * val,
// with an exact 0 for the plain ReLU.
template <int N>
__device__ __forceinline__ vd<N> vrelu(const vd<N> &x0, const vd<N> &val, double slope)
{
    vd<N> r;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        r.v[i] = x0.v[i] > 0. ? val.v[i] : (slope == 0. ? 0. : slope * val.v[i]);
    }
    return r;
}
#undef HY_VD_MAP1

template <int N>
__device__ __forceinline__ vd<N> vpow(const vd<N> &a, const vd<N> &b)
{
    vd<N> r;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        r.v[i] = ::pow(a.v[i], b.v[i]);
    }
    return r;
}

// pairwise_reduce() of up to 8 values (src/detail/llvm_helpers_algo.cpp:271-308), registers only.
template <int N>
__device__ __forceinline__ vd<N> pairwise8(vd<N> (&v)[8], std::uint32_t n)
{
    vd<N> w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        w[i] = (2 * i + 1 < static_cast<int>(n)) ? v[2 * i] + v[2 * i + 1] : v[2 * i];
    }
    const std::uint32_t m = (n + 1u) / 2u;
    vd<N> x[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        x[i] = (2 * i + 1 < static_cast<int>(m)) ? w[2 * i] + w[2 * i + 1] : w[2 * i];
    }
    const std::uint32_t m2 = (m + 1u) / 2u;
    return (m2 > 1u) ? x[0] + x[1] : x[0];
}

// sum_{j=j0..j1} A^[n-j] B^[j]. A and B are history rows: walked with two pointers (strides known at
// compile time, so the unrolled loop addresses with immediates).
template <int N, typename Row>
__device__ __forceinline__ vd<N> conv_plain(const Row &A, const Row &B, std::uint32_t n, std::uint32_t j0,
                                            std::uint32_t j1)
{
    vd<N> acc = splat<N>(0.);
    if (j1 + 1u > j0) {
        const double *pa = A.hptr(n - j0), *pb = B.hptr(j0);
        constexpr int S = static_cast<int>(Row::stride);
#pragma unroll 4
        for (std::uint32_t j = j0; j <= j1; ++j) {
            acc = vfma(Row::load(pa), Row::load(pb), acc);
            pa -= S;
            pb += S;
        }
    }
    return acc;
}

// sum_{j=j0..j1} j * (A^[n-j] B^[j]).
template <int N, typename Row>
__device__ __forceinline__ vd<N> conv_jw(const Row &A, const Row &B, std::uint32_t n, std::uint32_t j0,
                                         std::uint32_t j1)
{
    vd<N> acc = splat<N>(0.);
    if (j1 + 1u > j0) {
        const double *pa = A.hptr(n - j0), *pb = B.hptr(j0);
        constexpr int S = static_cast<int>(Row::stride);
#pragma unroll 4
        for (std::uint32_t j = j0; j <= j1; ++j) {
            acc = vfma(static_cast<double>(j), Row::load(pa) * Row::load(pb), acc);
            pa -= S;
            pb += S;
        }
    }
    return acc;
}

// Exponentiation by squaring with the reference's association order (src/math/pow.cpp:136-152).
template <int N>
__device__ inline vd<N> pow_ebs(vd<N> base, std::uint32_t e)
{
    vd<N> mult[6];
    int nm = 0;
    vd<N> b = base;
    while (e > 1u) {
        if (e & 1u) {
            mult[nm++] = b;
            e = (e - 1u) / 2u;
        } else {
            e /= 2u;
        }
        b = b * b;
    }
    vd<N> r = (e == 0u) ? splat<N>(1.) : b;
    for (int i = nm - 1; i >= 0; --i) {
        r = mult[i] * r;
    }
    return r;
}

// Order-0 evaluation of pow(x, expo) (src/math/pow.cpp:292-355).
template <int N>
__device__ inline vd<N> pow_eval(std::uint32_t algo, const vd<N> &x, const vd<N> &expo)
{
    const std::uint32_t type = algo >> 8, n = algo & 0xffu;
    switch (type) {
        case HY_POW_POS_SMALL_INT:
            return pow_ebs(x, n);
        case HY_POW_NEG_SMALL_INT:
            return 1. / pow_ebs(x, n);
        case HY_POW_POS_SMALL_HALF:
            return pow_ebs(vsqrt(x), n);
        case HY_POW_NEG_SMALL_HALF:
            return 1. / pow_ebs(vsqrt(x), n);
        default:
            return vpow(x, expo);
    }
}

__device__ inline std::uint32_t pow_algo_of(double e)
{
    if (isfinite(e) && e == trunc(e)) {
        if (e >= 0 && e <= 16) {
            return (HY_POW_POS_SMALL_INT << 8) | static_cast<std::uint32_t>(e);
        }
        if (e < 0 && -e <= 16) {
            return (HY_POW_NEG_SMALL_INT << 8) | static_cast<std::uint32_t>(-e);
        }
    } else if (isfinite(e)) {
        const double y = 2 * e;
        if (y == trunc(y)) {
            if (y >= 0 && y <= 16) {
                return (HY_POW_POS_SMALL_HALF << 8) | static_cast<std::uint32_t>(y);
            }
            if (y < 0 && -y <= 16) {
                return (HY_POW_NEG_SMALL_HALF << 8) | static_cast<std::uint32_t>(-y);
            }
        }
    }
    return HY_POW_GENERAL << 8;
}

// Value of a number/param reference (taylor_codegen_numparam, src/taylor_01.cpp:201-234).
template <int N, typename Tape>
__device__ __forceinline__ vd<N> numpar_val(const program &P, const Tape &t, std::uint32_t ref)
{
    return HY_REF_KIND(ref) == HY_REF_NUM ? splat<N>(t.cst(HY_REF_IDX(ref))) : t.par(HY_REF_IDX(ref));
}

// Functions whose arguments are all numbers/params: evaluated at order 0 only.
template <int N, typename Tape>
__device__ inline vd<N> cfunc_eval(const program &P, const Tape &t, std::uint32_t fn, std::uint32_t arg_off,
                                   std::uint32_t n)
{
    vd<N> v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        v[k] = (k < static_cast<int>(n)) ? numpar_val<N>(P, t, t.arg(arg_off + k)) : splat<N>(0.);
    }
    switch (fn) {
        case HY_CF_IDENTITY:
            return v[0];
        case HY_CF_SUM:
            return pairwise8(v, n);
        case HY_CF_PROD:
            return v[0] * v[1];
        case HY_CF_SUB:
            return v[0] - v[1];
        case HY_CF_DIV:
            return v[0] / v[1];
        case HY_CF_POW: {
            const std::uint32_t eref = t.arg(arg_off + 1u);
            const std::uint32_t algo
                = HY_REF_KIND(eref) == HY_REF_NUM ? pow_algo_of(v[1].v[0]) : (HY_POW_GENERAL << 8);
            return pow_eval(algo, v[0], v[1]);
        }
        case HY_CF_SUM_SQ:
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                v[k] = v[k] * v[k];
            }
            return pairwise8(v, n);
        case HY_CF_SIN:
            return vsin(v[0]);
        case HY_CF_COS:
            return vcos(v[0]);
        case HY_CF_TANH:
            return vtanh(v[0]);
        case HY_CF_EXP:
            return vexp(v[0]);
        case HY_CF_LOG:
            return vlog(v[0]);
        case HY_CF_SIGMOID:
            return vsigmoid(v[0]);
        case HY_CF_RELU:
            return vrelu(v[0], v[0], v[1].v[0]);
        case HY_CF_RELUP:
            return vrelup(v[0], v[1].v[0]);
    }
    return splat<N>(0.);
}

// Derivative of the (leaky) ReLU (src/math/relu.cpp:365-376): x > 0 ? 1 : slope.
template <int N>
__device__ __forceinline__ vd<N> vrelup(const vd<N> &x, double slope)
{
    vd<N> r;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        r.v[i] = x.v[i] > 0. ? 1. : slope;
    }
    return r;
}

// The order-n coefficient of the u variable defined by `op` (op.x = opcode, op.y/z/w = a/b/c operand
// fields). `self` is the row of the u variable being defined (read by the self-referential recurrences).
template <int N, typename Tape, typename Row>
__device__ __forceinline__ vd<N> diff_op(const program &P, const Tape &t, const uint4 &op, const Row &self,
                                         std::uint32_t n)
{
    using V = vd<N>;
    const std::uint32_t a = op.y, b = op.z, dep = op.w;

    switch (op.x) {
        case HY_OP_SUM: {
            // a^[n] = pairwise sum of the terms' order-n coefficients; numbers/params only at n = 0.
            V v[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                v[k] = splat<N>(0.);
                if (k < static_cast<int>(b)) {
                    const std::uint32_t ref = t.arg(a + k);
                    if (HY_REF_KIND(ref) == HY_REF_VAR) {
                        v[k] = t.row(HY_REF_IDX(ref)).at(n);
                    } else if (n == 0u) {
                        v[k] = numpar_val<N>(P, t, ref);
                    }
                }
            }
            return pairwise8(v, b);
        }
        case HY_OP_SUM_SQ: {
            // Per term the square recurrence, then a pairwise sum over the terms.
            V v[8];
            const bool odd = (n & 1u) != 0u;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                v[k] = splat<N>(0.);
                if (k < static_cast<int>(b)) {
                    const std::uint32_t ref = t.arg(a + k);
                    if (HY_REF_KIND(ref) == HY_REF_VAR) {
                        const Row A = t.row(HY_REF_IDX(ref));
                        if (odd) {
                            v[k] = conv_plain<N>(A, A, n, 0u, (n - 1u) / 2u);
                        } else {
                            const V ak2 = A.at(n / 2u);
                            const V sq = ak2 * ak2;
                            if (n > 0u) {
                                const V acc = conv_plain<N>(A, A, n, 0u, (n - 2u) / 2u);
                                v[k] = (acc + acc) + sq;
                            } else {
                                v[k] = sq;
                            }
                        }
                    } else if (n == 0u) {
                        const V val = numpar_val<N>(P, t, ref);
                        v[k] = val * val;
                    }
                }
            }
            const V r = pairwise8(v, b);
            return odd ? r + r : r;
        }
        case HY_OP_SUB_VV:
            return t.row(a).at(n) - t.row(b).at(n);
        case HY_OP_SUB_VN: {
            const V v = t.row(a).at(n);
            return n == 0u ? v - t.cst(b) : v;
        }
        case HY_OP_SUB_VP: {
            const V v = t.row(a).at(n);
            return n == 0u ? v - t.par(b) : v;
        }
        case HY_OP_SUB_NV: {
            const V v = t.row(b).at(n);
            return n == 0u ? t.cst(a) - v : -v;
        }
        case HY_OP_SUB_PV: {
            const V v = t.row(b).at(n);
            return n == 0u ? t.par(a) - v : -v;
        }
        case HY_OP_NEG:
            return -t.row(a).at(n);
        case HY_OP_MUL_NV:
            return t.cst(a) * t.row(b).at(n);
        case HY_OP_MUL_PV:
            return t.par(a) * t.row(b).at(n);
        case HY_OP_MUL_VV:
            // sum_{j=0..n} b^[n-j] c^[j]
            return conv_plain<N>(t.row(a), t.row(b), n, 0u, n);
        case HY_OP_DIV_VV:
        case HY_OP_DIV_NV:
        case HY_OP_DIV_PV: {
            // (b^[n] - sum_{j=1..n} a^[n-j] c^[j]) / c^[0], a = this u variable; numerator = -sum if b is constant.
            const Row C = t.row(b);
            const V c0 = C.at(0u);
            if (n == 0u) {
                const V num = op.x == HY_OP_DIV_VV ? t.row(a).at(0u)
                                                   : (op.x == HY_OP_DIV_NV ? splat<N>(t.cst(a)) : t.par(a));
                return num / c0;
            }
            const V acc = conv_plain<N>(self, C, n, 1u, n);
            if (op.x == HY_OP_DIV_VV) {
                return (t.row(a).at(n) - acc) / c0;
            }
            return (-acc) / c0;
        }
        case HY_OP_DIV_VN:
            return t.row(a).at(n) / t.cst(b);
        case HY_OP_DIV_VP:
            return t.row(a).at(n) / t.par(b);
        case HY_OP_SQUARE: {
            const Row A = t.row(a);
            if (n == 0u) {
                const V b0 = A.at(0u);
                return b0 * b0;
            }
            if (n & 1u) {
                const V r = conv_plain<N>(A, A, n, 0u, (n - 1u) / 2u);
                return r + r;
            }
            const V ak2 = A.at(n / 2u);
            const V sq = ak2 * ak2;
            const V r = conv_plain<N>(A, A, n, 0u, (n - 2u) / 2u);
            return (r + r) + sq;
        }
        case HY_OP_SQRT: {
            // (b^[n] - 2 sum_{j=1..} a^[n-j] a^[j] - [n even] (a^[n/2])^2) / (2 a^[0]), a = this u variable.
            if (n == 0u) {
                return vsqrt(t.row(a).at(0u));
            }
            V div = self.at(0u);
            div = div + div;
            V fac = t.row(a).at(n);
            const bool even = (n & 1u) == 0u;
            const std::uint32_t upper = (n - (even ? 2u : 1u)) / 2u;
            V acc = conv_plain<N>(self, self, n, 1u, upper);
            acc = acc + acc;
            if (even) {
                const V tmp = self.at(n / 2u);
                fac = fac - tmp * tmp;
            }
            fac = fac - acc;
            return fac / div;
        }
        case HY_OP_POW_VN:
        case HY_OP_POW_VP: {
            // (1 / (n b0)) sum_{j=0..n-1} [n alpha - j (alpha + 1)] b^[n-j] a^[j], a = this u variable.
            const V alpha = op.x == HY_OP_POW_VN ? splat<N>(t.cst(b)) : t.par(b);
            const Row B = t.row(a);
            if (n == 0u) {
                return pow_eval(op.x == HY_OP_POW_VN ? dep : (HY_POW_GENERAL << 8), B.at(0u), alpha);
            }
            const double nd = static_cast<double>(n);
            const V ap1 = alpha + 1.;
            const V n_alpha = nd * alpha;
            V acc = splat<N>(0.);
            const double *pb = B.hptr(n), *pa = self.hptr(0u);
            constexpr int S = static_cast<int>(Row::stride);
#pragma unroll 4
            for (std::uint32_t j = 0; j < n; ++j) {
                const V fac = n_alpha - static_cast<double>(j) * ap1;
                acc = vfma(fac, Row::load(pb) * Row::load(pa), acc);
                pb -= S;
                pa += S;
            }
            return acc / (nd * B.at(0u));
        }
        case HY_OP_SIN:
            // (1/n) sum_{j=1..n} j c^[n-j] b^[j], c = cosine of b (hidden dependency).
            if (n == 0u) {
                return vsin(t.row(a).at(0u));
            }
            return conv_jw<N>(t.row(dep), t.row(a), n, 1u, n) / static_cast<double>(n);
        case HY_OP_COS:
            // sum / (-n), with s = sine of b as hidden dependency.
            if (n == 0u) {
                return vcos(t.row(a).at(0u));
            }
            return conv_jw<N>(t.row(dep), t.row(a), n, 1u, n) / (-static_cast<double>(n));
        case HY_OP_TANH: {
            // b^[n] - (1/n) sum_{j=1..n} j c^[n-j] b^[j], c = tanh(b)^2 (hidden dependency).
            const Row B = t.row(a);
            if (n == 0u) {
                return vtanh(B.at(0u));
            }
            return B.at(n) - conv_jw<N>(t.row(dep), B, n, 1u, n) / static_cast<double>(n);
        }
        case HY_OP_EXP:
            // (1/n) sum_{j=1..n} j a^[n-j] b^[j], a = this u variable.
            if (n == 0u) {
                return vexp(t.row(a).at(0u));
            }
            return conv_jw<N>(self, t.row(a), n, 1u, n) / static_cast<double>(n);
        case HY_OP_LOG: {
            // (n b^[n] - sum_{j=1..n-1} j b^[n-j] a^[j]) / (n b^[0]), a = this u variable.
            const Row B = t.row(a);
            if (n == 0u) {
                return vlog(B.at(0u));
            }
            const double nd = static_cast<double>(n);
            const V nb0 = nd * B.at(0u);
            V ret = nd * B.at(n);
            if (n > 1u) {
                ret = ret - conv_jw<N>(B, self, n, 1u, n - 1u);
            }
            return ret / nb0;
        }
        case HY_OP_TIME:
            return n == 0u ? t.time() : (n == 1u ? splat<N>(1.) : splat<N>(0.));
        case HY_OP_CFUNC:
            return n == 0u ? cfunc_eval<N>(P, t, a, b, dep) : splat<N>(0.);
        case HY_OP_SIGMOID: {
            // (1/n) sum_{j=1..n} j (a^[n-j] - c^[n-j]) b^[j], a = this u variable, c = a^2 (hidden dependency).
            const Row B = t.row(a);
            if (n == 0u) {
                return vsigmoid(B.at(0u));
            }
            const Row C = t.row(dep);
            V acc = splat<N>(0.);
            constexpr int S = static_cast<int>(Row::stride);
            const double *pa = self.hptr(n - 1u), *pc = C.hptr(n - 1u), *pb = B.hptr(1u);
            for (std::uint32_t j = 1; j <= n; ++j) {
                acc = vfma(static_cast<double>(j), (Row::load(pa) - Row::load(pc)) * Row::load(pb), acc);
                pa -= S;
                pc -= S;
                pb += S;
            }
            return acc / static_cast<double>(n);
        }
        case HY_OP_RELU: {
            const Row B = t.row(a);
            return vrelu(B.at(0u), B.at(n), t.cst(b));
        }
        case HY_OP_RELUP:
            // Piecewise constant: relup at order 0, zero afterwards (src/math/relu.cpp:404-424).
            return n == 0u ? vrelup(t.row(a).at(0u), t.cst(b)) : splat<N>(0.);
    }
    return splat<N>(0.);
}

// x / n for a small positive integer n, correctly rounded, without the ~35-instruction IEEE division
// routine: q = RN(x * RN(1/n)), r = x - q n (exact, by fma), q' = RN(q + r RN(1/n)) (Markstein's correction
// step; verified against true division on 1.9e9 random and integer-valued inputs for n = 1..64). Outside the
// range where the residual is guaranteed exact (tiny / huge / non-finite x) the true division is used.
__device__ __forceinline__ double div_small_int(double x, std::uint32_t n)
{
    const double nd = static_cast<double>(n);
    const double ax = fabs(x);
    if (n > 64u || !(ax > 0x1p-900 && ax < 0x1p900)) {
        return x / nd;
    }
    const double y = 1. / nd; // n is warp-uniform: one division per warp and order at most (hoisted by callers)
    const double q = x * y;
    const double r = ::fma(-q, nd, x);
    return ::fma(r, y, q);
}
// The (cold) IEEE division fallback, kept out of line: the division routine is ~40 instructions and would be
// inlined at every call site otherwise.
static __device__ __noinline__ double div_fallback(double x, double nd)
{
    return x / nd;
}
template <int N>
__device__ __forceinline__ vd<N> div_small_int(const vd<N> &x, std::uint32_t n, double nd, double rcp)
{
    vd<N> out;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const double ax = fabs(x.v[i]);
        if (n > 64u || !(ax > 0x1p-900 && ax < 0x1p900)) {
            out.v[i] = div_fallback(x.v[i], nd);
        } else {
            const double q = x.v[i] * rcp;
            const double r = ::fma(-q, nd, x.v[i]);
            out.v[i] = ::fma(r, rcp, q);
        }
    }
    return out;
}

// Order-n (n >= 1) coefficient of a state variable whose first derivative is `ref`: (u_rhs)^[n-1] / n, a true
// division in the reference (src/taylor_02.cpp:245-287), computed here by div_small_int() (same result);
// constant right-hand sides only contribute at n == 1. nd = (double)n, rcp = 1 / nd.
template <int N, typename Tape>
__device__ __forceinline__ vd<N> sv_diff(const program &P, const Tape &t, std::uint32_t ref, std::uint32_t n, double nd,
                                         double rcp)
{
    if (HY_REF_KIND(ref) == HY_REF_VAR) {
        return div_small_int(t.row(HY_REF_IDX(ref)).at(n - 1u), n, nd, rcp);
    }
    return n == 1u ? numpar_val<N>(P, t, ref) : splat<N>(0.);
}

// std::max / std::min semantics of the reference's llvm_max/llvm_min (src/detail/llvm_helpers_cmp.cpp:313-329).
__device__ __forceinline__ double std_max(double a, double b)
{
    return (a < b) ? b : a;
}
__device__ __forceinline__ double std_min(double a, double b)
{
    return (b < a) ? b : a;
}

// taylor_determine_h() (src/taylor_00.cpp:102-273) from the three infinity norms: Jorba-Zou step size,
// clamped to |max_delta_t|, signed like max_delta_t.
// (The program's three constants as values: for out-of-line callers, which would otherwise copy the program to
// local memory to pass it by reference.)
__device__ __forceinline__ double h_from_norms(double inv_p, double inv_pm1, double rhofac, double m0, double mp,
                                               double mp1, double max_delta_t)
{
    const double num_rho = (m0 <= 1.) ? 1. : m0;
    const double rho_o = ::pow(num_rho / mp, inv_p);
    const double rho_om1 = ::pow(num_rho / mp1, inv_pm1);
    const double rho_m = std_min(rho_o, rho_om1);
    double h = rho_m * rhofac;
    h = std_min(h, fabs(max_delta_t));
    return (max_delta_t < 0.) ? -h : h;
}
__device__ __forceinline__ double h_from_norms(const program &P, double m0, double mp, double mp1, double max_delta_t)
{
    return h_from_norms(P.inv_p, P.inv_pm1, P.rhofac, m0, mp, mp1, max_delta_t);
}

// Evaluation of one Taylor polynomial at h: Horner (src/taylor_00.cpp:279-351) or compensated summation of
// the monomials (src/taylor_00.cpp:355-460) when high_accuracy. cf(o) returns the order-o coefficient.
template <typename F>
__device__ __forceinline__ double eval_poly(const program &P, const F &cf, double h)
{
    const std::uint32_t p = P.order;
    double res;
    if (!P.high_accuracy) {
        res = cf(p);
        for (std::uint32_t o = 1; o <= p; ++o) {
            res = ::fma(res, h, cf(p - o));
        }
    } else {
        res = cf(0u);
        double comp = 0., cur_h = h;
        for (std::uint32_t o = 1; o <= p; ++o) {
            const double tmp = __dmul_rn(cf(o), cur_h);
            const double y = __dsub_rn(tmp, comp);
            const double tt = __dadd_rn(res, y);
            comp = __dsub_rn(__dsub_rn(tt, res), y);
            res = tt;
            cur_h = __dmul_rn(cur_h, h);
        }
    }
    return res;
}

// K polynomials evaluated side by side (same operations per polynomial as eval_poly(); the K chains are
// independent, so that the loads of their coefficients overlap). c[k] points to the order-0 coefficient,
// consecutive orders are `stride` doubles apart.
template <int K>
__device__ __forceinline__ void eval_poly_k(const program &P, const double *const (&c)[K], std::size_t stride, double h,
                                            double (&res)[K])
{
    const std::uint32_t p = P.order;
    if (!P.high_accuracy) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
            res[k] = c[k][static_cast<std::size_t>(p) * stride];
        }
        for (std::uint32_t o = 1; o <= p; ++o) {
#pragma unroll
            for (int k = 0; k < K; ++k) {
                res[k] = ::fma(res[k], h, c[k][static_cast<std::size_t>(p - o) * stride]);
            }
        }
    } else {
        double comp[K], cur_h = h;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            res[k] = c[k][0];
            comp[k] = 0.;
        }
        for (std::uint32_t o = 1; o <= p; ++o) {
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const double tmp = __dmul_rn(c[k][static_cast<std::size_t>(o) * stride], cur_h);
                const double y = __dsub_rn(tmp, comp[k]);
                const double tt = __dadd_rn(res[k], y);
                comp[k] = __dsub_rn(__dsub_rn(tt, res[k]), y);
                res[k] = tt;
            }
            cur_h = __dmul_rn(cur_h, h);
        }
    }
}

// Double-length time arithmetic (include/heyoka/detail/dfloat.hpp:104-169).
struct dfl {
    double hi, lo;
};

__device__ __forceinline__ dfl eft_knuth(double a, double b)
{
    const double x = __dadd_rn(a, b);
    const double z = __dsub_rn(x, a);
    const double y = __dadd_rn(__dsub_rn(a, __dsub_rn(x, z)), __dsub_rn(b, z));
    return {x, y};
}
__device__ __forceinline__ dfl eft_dekker(double a, double b)
{
    const double x = __dadd_rn(a, b);
    const double y = __dadd_rn(__dsub_rn(a, x), b);
    return {x, y};
}
__device__ __forceinline__ dfl dfl_add(dfl a, dfl b)
{
    const dfl h = eft_knuth(a.hi, b.hi);
    const dfl l = eft_knuth(a.lo, b.lo);
    dfl uv = eft_dekker(h.hi, __dadd_rn(h.lo, l.hi));
    uv = eft_dekker(uv.hi, __dadd_rn(uv.lo, l.lo));
    return uv;
}
__device__ __forceinline__ dfl dfl_sub(dfl a, dfl b)
{
    return dfl_add(a, dfl{-b.hi, -b.lo});
}
__device__ __forceinline__ bool dfl_lt(dfl x, dfl y)
{
    return (x.hi < y.hi) || (x.hi == y.hi && x.lo < y.lo);
}
__device__ __forceinline__ bool dfl_ge0(dfl x)
{
    return (x.hi > 0.) || (x.hi == 0. && x.lo >= 0.);
}

// Time limit of a propagate_until() step (src/taylor_adaptive_batch.cpp:1378-1387).
__device__ __forceinline__ double step_limit(bool dir, dfl rem, double mdt)
{
    const dfl lim = dir ? (dfl_lt(rem, dfl{mdt, 0.}) ? rem : dfl{mdt, 0.})
                        : (dfl_lt(rem, dfl{-mdt, 0.}) ? dfl{-mdt, 0.} : rem);
    return lim.hi;
}

} // namespace heyoka_b200::dev

#endif
