/* TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * CPU oracle for the batch Taylor hot path: a plain-C restatement of what heyoka's JIT-compiled
 * stepper computes (bluescarni/heyoka @ 9c91f71), driven by the same lowered program
 * (hy_program_desc, include/heyoka_b200.h) that the CUDA kernels interpret. Only tests/,
 * __graft_entry__.smoke() and bench.py's CPU-baseline legs may load this library; the product
 * (heyoka_b200/) never links or calls it.
 *
 * Parity status: PINNED. The reference cannot be built in this image (LLVM 18-22 dev libraries,
 * Boost >= 1.85, fmt, spdlog, oneTBB are absent), so this restatement is checked against the
 * reference's own known answers: the closed-form jets of test/taylor_*.cpp, the step-size formula
 * of test/timestep_check.cpp, the printed outputs of doc/tut_batch_mode.rst and README.md, and the
 * exact step counts of test/taylor_adaptive_batch.cpp:586-598, and the outputs printed in doc/tut_adaptive.rst,
 * tut_d_output.rst, tut_ensemble.rst, tut_param.rst, tut_nonauto.rst, tut_adaptive_custom.rst and tut_events.rst (states
 * to the 16-17 printed digits, exact step counts, event times to an ulp; see tests/test_oracle_golden.py,
 * tests/test_events_cpu.py).
 *
 * What follows what:
 *   jet evaluation order            src/taylor_02.cpp:1339-1418 (default mode), :1147-1185 (compact)
 *   state-variable derivatives      src/taylor_02.cpp:245-287
 *   sum / sub                       src/math/sum.cpp:185-238, src/detail/sub.cpp:64-124
 *   prod (k*v, -v, v*v)             src/math/prod.cpp:316-396 (pairwise), :640-698 (sequential)
 *   div                             src/detail/div.cpp:64-147, :189-431
 *   square / sqrt / pow             src/math/pow.cpp:390-550, :618-963; order-0 algo :292-355, :136-152
 *   sum_sq                          src/detail/sum_sq.cpp:100-245, :250-468
 *   sin / cos / tanh / exp / log    src/math/sin.cpp:152-190, cos.cpp:152-190, tanh.cpp:111-149,
 *                                   exp.cpp:75-112, log.cpp:78-127
 *   time, all-constant functions    src/math/time.cpp:82-104, include/heyoka/detail/taylor_common.hpp:88-157
 *   step size                       src/taylor_00.cpp:84-94, :102-273; max/min = std::max/min
 *                                   (src/detail/llvm_helpers_cmp.cpp:313-329)
 *   state update                    src/taylor_00.cpp:279-351 (Horner), :355-460 (compensated)
 *   tc layout                       src/taylor_00.cpp:574-580
 *   step bookkeeping                src/taylor_adaptive_batch.cpp:632-727
 *   propagate_until loop            src/taylor_adaptive_batch.cpp:1256-1273, :1372-1527
 *   double-length time              include/heyoka/detail/dfloat.hpp:104-169
 *
 * Two summation orders exist in the reference and both are restated, selectable at run time:
 *   ORACLE_PAIRWISE   default (non-compact) mode: products collected, then pairwise_sum
 *                     (src/detail/llvm_helpers_algo.cpp:271-308)
 *   sequential        compact mode: running accumulator
 * and ORACLE_FMA fuses `acc + a*b` into fma(a, b, acc) in sequential mode, which is one of the
 * contractions LLVM is allowed to perform (src/llvm_state.cpp:842-845) and the one the CUDA
 * kernels use. The scalar build (ORACLE_W == 1) is compiled with -ffp-contract=off so that every
 * rounding is explicit. The ORACLE_W == 8 build processes 8 lanes per call with GCC vector
 * extensions and -ffp-contract=fast -march=native: it is the timed "CPU port" baseline.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/heyoka_b200.h"

#ifndef ORACLE_W
#define ORACLE_W 1
#endif

#define ORACLE_PAIRWISE 1
#define ORACLE_FMA 2
/* ORACLE_W != 1 only: run the per-lane scalar tail (step size, state update) instead of the SIMD one (A/B check). */
#define ORACLE_SCALAR_TAIL 4

#if ORACLE_W == 1
typedef double real_t;
#define R_GET(v, l) (v)
#define R_SET(v, l, x) ((v) = (x))
#define R_SPLAT(x) (x)
#define SYM(name) name##_w1
#else
typedef double real_t __attribute__((vector_size(ORACLE_W * 8), aligned(8)));
#define R_GET(v, l) ((v)[l])
#define R_SET(v, l, x) ((v)[l] = (x))
#define R_SPLAT(x) (((real_t){0} + (x)))
#define SYM3(name, w) name##_w##w
#define SYM2(name, w) SYM3(name, w)
#define SYM(name) SYM2(name, ORACLE_W)
#endif

#define MAX_NARY 64

typedef struct {
    const hy_program_desc *P;
    uint32_t batch;   /* stride of the external arrays */
    uint32_t lane0;   /* first lane of this group */
    uint32_t nl;      /* valid lanes in this group (<= ORACLE_W) */
    const double *pars;
    real_t *T; /* tape: T[o * n_uvars + u]; followed by 3 * n_eq vectors of scratch (alloc_tape()) */
    int mode;
} ctx_t;

/* ---- helpers -------------------------------------------------------------------------------- */

static inline real_t r_fma(const ctx_t *c, real_t a, real_t b, real_t acc)
{
#if ORACLE_W == 1
    if (c->mode & ORACLE_FMA) {
        return fma(a, b, acc);
    }
    return acc + a * b;
#else
    (void)c;
    return acc + a * b; /* contracted by the compiler (-ffp-contract=fast) */
#endif
}

static inline real_t r_sqrt(real_t x)
{
#if ORACLE_W == 1
    return sqrt(x);
#else
    real_t r;
    for (int l = 0; l < ORACLE_W; ++l) {
        r[l] = sqrt(x[l]);
    }
    return r;
#endif
}

#define R_MAP1(fn, x, out)                                                                                             \
    do {                                                                                                               \
        for (int l_ = 0; l_ < ORACLE_W; ++l_) {                                                                        \
            R_SET(out, l_, fn(R_GET(x, l_)));                                                                          \
        }                                                                                                              \
    } while (0)

/* src/math/sigmoid.cpp:69-75; src/math/relu.cpp:118-128 (gate on x0, exact 0 for the plain ReLU). */
static inline double sigmoid_d(double x)
{
    return 1. / (1. + exp(-x));
}
static inline double relu_d(double x0, double val, double slope)
{
    return x0 > 0. ? val : (slope == 0. ? 0. : slope * val);
}

static inline real_t r_pow(real_t x, real_t y)
{
    real_t r = R_SPLAT(0.);
    for (int l = 0; l < ORACLE_W; ++l) {
        R_SET(r, l, pow(R_GET(x, l), R_GET(y, l)));
    }
    return r;
}

/* pairwise_reduce with fadd (src/detail/llvm_helpers_algo.cpp:271-308). In place; n >= 1. */
static real_t pairwise_sum(real_t *v, uint32_t n)
{
    while (n != 1u) {
        uint32_t m = 0;
        for (uint32_t i = 0; i < n; i += 2u) {
            if (i + 1u == n) {
                v[m++] = v[i];
            } else {
                v[m++] = v[i] + v[i + 1u];
            }
        }
        n = m;
    }
    return v[0];
}

static inline real_t load_par(const ctx_t *c, uint32_t idx)
{
    real_t r = R_SPLAT(0.);
    for (uint32_t l = 0; l < ORACLE_W; ++l) {
        const uint32_t ll = l < c->nl ? l : c->nl - 1u;
        R_SET(r, l, c->pars[(size_t)idx * c->batch + c->lane0 + ll]);
    }
    return r;
}

/* Value of a number/param reference (taylor_codegen_numparam, src/taylor_01.cpp:201-234). */
static inline real_t numpar_val(const ctx_t *c, uint32_t ref)
{
    if (HY_REF_KIND(ref) == HY_REF_NUM) {
        return R_SPLAT(c->P->consts[HY_REF_IDX(ref)]);
    }
    return load_par(c, HY_REF_IDX(ref));
}

#define TAPE(c, o, u) ((c)->T[(size_t)(o) * (c)->P->n_uvars + (u)])

/* Exponentiation by squaring (src/math/pow.cpp:136-152). */
static real_t pow_ebs(real_t base, uint32_t e)
{
    if (e == 0u) {
        return R_SPLAT(1.);
    }
    if (e == 1u) {
        return base;
    }
    if (e % 2u == 0u) {
        return pow_ebs(base * base, e / 2u);
    }
    return base * pow_ebs(base * base, (e - 1u) / 2u);
}

/* Order-0 evaluation of pow(x, expo) (src/math/pow.cpp:292-355). */
static real_t pow_eval(uint32_t algo, real_t x, real_t expo)
{
    const uint32_t type = algo >> 8, n = algo & 0xffu;
    switch (type) {
        case HY_POW_POS_SMALL_INT:
            return pow_ebs(x, n);
        case HY_POW_NEG_SMALL_INT:
            return R_SPLAT(1.) / pow_ebs(x, n);
        case HY_POW_POS_SMALL_HALF:
            return pow_ebs(r_sqrt(x), n);
        case HY_POW_NEG_SMALL_HALF:
            return R_SPLAT(1.) / pow_ebs(r_sqrt(x), n);
        default:
            return r_pow(x, expo);
    }
}

static uint32_t pow_algo_of(double e)
{
    /* get_pow_eval_algo(), src/math/pow.cpp:292-355 (restated independently of the product's lowering). */
    if (isfinite(e) && e == trunc(e)) {
        if (e >= 0 && e <= 16) {
            return (HY_POW_POS_SMALL_INT << 8) | (uint32_t)e;
        }
        if (e < 0 && -e <= 16) {
            return (HY_POW_NEG_SMALL_INT << 8) | (uint32_t)(-e);
        }
    } else if (isfinite(e)) {
        const double y = 2 * e;
        if (y == trunc(y)) {
            if (y >= 0 && y <= 16) {
                return (HY_POW_POS_SMALL_HALF << 8) | (uint32_t)y;
            }
            if (y < 0 && -y <= 16) {
                return (HY_POW_NEG_SMALL_HALF << 8) | (uint32_t)(-y);
            }
        }
    }
    return HY_POW_GENERAL << 8;
}

/* Functions of constants only: value at order 0, zero afterwards. */
static real_t cfunc_eval(const ctx_t *c, const hy_op *op)
{
    real_t v[MAX_NARY];
    const uint32_t n = op->c;
    for (uint32_t k = 0; k < n; ++k) {
        v[k] = numpar_val(c, c->P->args[op->b + k]);
    }
    real_t r = R_SPLAT(0.);
    switch (op->a) {
        case HY_CF_IDENTITY:
            return v[0];
        case HY_CF_SUM:
            return pairwise_sum(v, n);
        case HY_CF_PROD:
            /* -1 * x is a negation (src/math/prod.cpp:321-338). */
            return v[0] * v[1];
        case HY_CF_SUB:
            return v[0] - v[1];
        case HY_CF_DIV:
            return v[0] / v[1];
        case HY_CF_POW: {
            /* The algorithm is selected from the exponent when it is a number. */
            const uint32_t eref = c->P->args[op->b + 1u];
            const uint32_t algo
                = HY_REF_KIND(eref) == HY_REF_NUM ? pow_algo_of(c->P->consts[HY_REF_IDX(eref)]) : (HY_POW_GENERAL << 8);
            return pow_eval(algo, v[0], v[1]);
        }
        case HY_CF_SUM_SQ:
            for (uint32_t k = 0; k < n; ++k) {
                v[k] = v[k] * v[k];
            }
            return pairwise_sum(v, n);
        case HY_CF_SIN:
            R_MAP1(sin, v[0], r);
            return r;
        case HY_CF_COS:
            R_MAP1(cos, v[0], r);
            return r;
        case HY_CF_TANH:
            R_MAP1(tanh, v[0], r);
            return r;
        case HY_CF_EXP:
            R_MAP1(exp, v[0], r);
            return r;
        case HY_CF_LOG:
            R_MAP1(log, v[0], r);
            return r;
        case HY_CF_SIGMOID:
            R_MAP1(sigmoid_d, v[0], r);
            return r;
        case HY_CF_RELU:
            for (int l_ = 0; l_ < ORACLE_W; ++l_) {
                R_SET(r, l_, relu_d(R_GET(v[0], l_), R_GET(v[0], l_), R_GET(v[1], l_)));
            }
            return r;
        case HY_CF_RELUP:
            for (int l_ = 0; l_ < ORACLE_W; ++l_) {
                R_SET(r, l_, R_GET(v[0], l_) > 0. ? 1. : R_GET(v[1], l_));
            }
            return r;
    }
    return r;
}

/* Generic "sum_j w(j) * A[n-j] * B[j]" accumulation in the two summation orders.
 * weight == 0: plain products; weight == 1: j * (a*b) (sin/cos/tanh/exp/log);
 * weight == 2: (n*alpha - j*(alpha+1)) * (a*b) (pow). j runs over [j0, j1]. */
static real_t conv(const ctx_t *c, uint32_t n, uint32_t ua, uint32_t ub, uint32_t j0, uint32_t j1, int weight,
                   real_t alpha)
{
    real_t buf[256];
    real_t acc = R_SPLAT(0.);
    uint32_t cnt = 0;
    if (j1 < j0 || j1 == (uint32_t)-1) {
        return acc;
    }
    for (uint32_t j = j0; j <= j1; ++j) {
        const real_t a = TAPE(c, n - j, ua), b = TAPE(c, j, ub);
        if (c->mode & ORACLE_PAIRWISE) {
            real_t t = a * b;
            if (weight == 1) {
                t = R_SPLAT((double)j) * t;
            } else if (weight == 2) {
                const real_t fac = R_SPLAT((double)n) * alpha - R_SPLAT((double)j) * (alpha + R_SPLAT(1.));
                t = fac * t;
            }
            buf[cnt++] = t;
        } else {
            if (weight == 0) {
                acc = r_fma(c, a, b, acc);
            } else if (weight == 1) {
                acc = r_fma(c, R_SPLAT((double)j), a * b, acc);
            } else {
                const real_t fac = R_SPLAT((double)n) * alpha - R_SPLAT((double)j) * (alpha + R_SPLAT(1.));
                acc = r_fma(c, fac, a * b, acc);
            }
        }
    }
    if (c->mode & ORACLE_PAIRWISE) {
        return cnt ? pairwise_sum(buf, cnt) : R_SPLAT(0.);
    }
    return acc;
}

/* ---- one u variable at one order ------------------------------------------------------------ */
static real_t diff_op(const ctx_t *c, const hy_op *op, uint32_t u_idx, uint32_t n, real_t time_v)
{
    const hy_program_desc *P = c->P;
    const real_t zero = R_SPLAT(0.);
    real_t r = zero;

    switch (op->opcode) {
        case HY_OP_SUM: {
            real_t v[MAX_NARY];
            for (uint32_t k = 0; k < op->b; ++k) {
                const uint32_t ref = P->args[op->a + k];
                if (HY_REF_KIND(ref) == HY_REF_VAR) {
                    v[k] = TAPE(c, n, HY_REF_IDX(ref));
                } else {
                    v[k] = n == 0u ? numpar_val(c, ref) : zero;
                }
            }
            return pairwise_sum(v, op->b);
        }
        case HY_OP_SUM_SQ: {
            const uint32_t nt = op->b;
            real_t tmp[MAX_NARY];
            if (n % 2u == 1u) {
                const uint32_t jmax = (n - 1u) / 2u;
                for (uint32_t k = 0; k < nt; ++k) {
                    const uint32_t ref = P->args[op->a + k];
                    tmp[k] = HY_REF_KIND(ref) == HY_REF_VAR ? conv(c, n, HY_REF_IDX(ref), HY_REF_IDX(ref), 0, jmax, 0, zero)
                                                            : zero;
                }
                r = pairwise_sum(tmp, nt);
                return r + r;
            }
            for (uint32_t k = 0; k < nt; ++k) {
                const uint32_t ref = P->args[op->a + k];
                real_t sq;
                if (HY_REF_KIND(ref) == HY_REF_VAR) {
                    const real_t ak2 = TAPE(c, n / 2u, HY_REF_IDX(ref));
                    sq = ak2 * ak2;
                } else if (n == 0u) {
                    const real_t val = numpar_val(c, ref);
                    sq = val * val;
                } else {
                    sq = zero;
                }
                if (n > 0u) {
                    real_t acc = HY_REF_KIND(ref) == HY_REF_VAR
                                     ? conv(c, n, HY_REF_IDX(ref), HY_REF_IDX(ref), 0, (n - 2u) / 2u, 0, zero)
                                     : zero;
                    acc = acc + acc;
                    tmp[k] = acc + sq;
                } else {
                    tmp[k] = sq;
                }
            }
            return pairwise_sum(tmp, nt);
        }
        case HY_OP_SUB_VV:
            return TAPE(c, n, op->a) - TAPE(c, n, op->b);
        case HY_OP_SUB_VN:
        case HY_OP_SUB_VP: {
            const real_t v = TAPE(c, n, op->a);
            if (n == 0u) {
                return v - numpar_val(c, HY_REF(op->opcode == HY_OP_SUB_VN ? HY_REF_NUM : HY_REF_PAR, op->b));
            }
            return v;
        }
        case HY_OP_SUB_NV:
        case HY_OP_SUB_PV: {
            const real_t v = TAPE(c, n, op->b);
            if (n == 0u) {
                return numpar_val(c, HY_REF(op->opcode == HY_OP_SUB_NV ? HY_REF_NUM : HY_REF_PAR, op->a)) - v;
            }
            return -v;
        }
        case HY_OP_NEG:
            return -TAPE(c, n, op->a);
        case HY_OP_MUL_NV:
            return R_SPLAT(P->consts[op->a]) * TAPE(c, n, op->b);
        case HY_OP_MUL_PV:
            return load_par(c, op->a) * TAPE(c, n, op->b);
        case HY_OP_MUL_VV:
            /* sum_{j=0..n} b^[n-j] c^[j]. */
            return conv(c, n, op->a, op->b, 0, n, 0, zero);
        case HY_OP_DIV_VV:
        case HY_OP_DIV_NV:
        case HY_OP_DIV_PV: {
            const real_t c0 = TAPE(c, 0, op->b);
            if (n == 0u) {
                const real_t num = op->opcode == HY_OP_DIV_VV
                                       ? TAPE(c, 0, op->a)
                                       : numpar_val(c, HY_REF(op->opcode == HY_OP_DIV_NV ? HY_REF_NUM : HY_REF_PAR, op->a));
                return num / c0;
            }
            /* sum_{j=1..n} a^[n-j] c^[j], a = this u variable. The sequential (compact-mode) form
             * multiplies c^[j] * a^[n-j]; multiplication commutes, so the rounding is the same. */
            const real_t acc = conv(c, n, u_idx, op->b, 1, n, 0, zero);
            if (op->opcode == HY_OP_DIV_VV) {
                return (TAPE(c, n, op->a) - acc) / c0;
            }
            return (-acc) / c0;
        }
        case HY_OP_DIV_VN:
            return TAPE(c, n, op->a) / R_SPLAT(P->consts[op->b]);
        case HY_OP_DIV_VP:
            return TAPE(c, n, op->a) / load_par(c, op->b);
        case HY_OP_SQUARE: {
            if (n == 0u) {
                const real_t b0 = TAPE(c, 0, op->a);
                return b0 * b0;
            }
            if (n % 2u == 1u) {
                r = conv(c, n, op->a, op->a, 0, (n - 1u) / 2u, 0, zero);
                return r + r;
            }
            const real_t ak2 = TAPE(c, n / 2u, op->a);
            const real_t sq = ak2 * ak2;
            r = conv(c, n, op->a, op->a, 0, (n - 2u) / 2u, 0, zero);
            return (r + r) + sq;
        }
        case HY_OP_SQRT: {
            if (n == 0u) {
                return r_sqrt(TAPE(c, 0, op->a));
            }
            real_t div = TAPE(c, 0, u_idx);
            div = div + div;
            real_t fac = TAPE(c, n, op->a);
            const int even = (n % 2u == 0u);
            const uint32_t upper = (n - (even ? 2u : 1u)) / 2u;
            if (c->mode & ORACLE_PAIRWISE) {
                /* src/math/pow.cpp:432-480: the a^[n/2]^2 term is subtracted first, then 2*sum. */
                if (even) {
                    const real_t t = TAPE(c, n / 2u, u_idx);
                    fac = fac - t * t;
                }
                if (upper >= 1u) {
                    real_t s = conv(c, n, u_idx, u_idx, 1, upper, 0, zero);
                    s = s + s;
                    fac = fac - s;
                }
                return fac / div;
            }
            /* src/math/pow.cpp:735-845 (compact mode): acc doubled, then the square, then acc. */
            real_t acc = upper >= 1u ? conv(c, n, u_idx, u_idx, 1, upper, 0, zero) : zero;
            acc = acc + acc;
            if (even) {
                const real_t t = TAPE(c, n / 2u, u_idx);
                fac = fac - t * t;
            }
            fac = fac - acc;
            return fac / div;
        }
        case HY_OP_POW_VN:
        case HY_OP_POW_VP: {
            const real_t alpha = op->opcode == HY_OP_POW_VN ? R_SPLAT(P->consts[op->b]) : load_par(c, op->b);
            if (n == 0u) {
                return pow_eval(op->opcode == HY_OP_POW_VN ? op->c : (HY_POW_GENERAL << 8), TAPE(c, 0, op->a), alpha);
            }
            /* (1 / (n b0)) sum_{j=0..n-1} [n alpha - j (alpha + 1)] b^[n-j] a^[j]. */
            const real_t acc = conv(c, n, op->a, u_idx, 0, n - 1u, 2, alpha);
            return acc / (R_SPLAT((double)n) * TAPE(c, 0, op->a));
        }
        case HY_OP_SIN: {
            if (n == 0u) {
                R_MAP1(sin, TAPE(c, 0, op->a), r);
                return r;
            }
            /* (1/n) sum_{j=1..n} j c^[n-j] b^[j], c = cos(b). */
            return conv(c, n, op->c, op->a, 1, n, 1, zero) / R_SPLAT((double)n);
        }
        case HY_OP_COS: {
            if (n == 0u) {
                R_MAP1(cos, TAPE(c, 0, op->a), r);
                return r;
            }
            /* sum / (-n), s = sin(b). */
            return conv(c, n, op->c, op->a, 1, n, 1, zero) / R_SPLAT(-(double)n);
        }
        case HY_OP_TANH: {
            if (n == 0u) {
                R_MAP1(tanh, TAPE(c, 0, op->a), r);
                return r;
            }
            /* b^[n] - (1/n) sum_{j=1..n} j c^[n-j] b^[j], c = tanh(b)^2. */
            return TAPE(c, n, op->a) - conv(c, n, op->c, op->a, 1, n, 1, zero) / R_SPLAT((double)n);
        }
        case HY_OP_EXP: {
            if (n == 0u) {
                R_MAP1(exp, TAPE(c, 0, op->a), r);
                return r;
            }
            /* (1/n) sum_{j=1..n} j a^[n-j] b^[j]. */
            return conv(c, n, u_idx, op->a, 1, n, 1, zero) / R_SPLAT((double)n);
        }
        case HY_OP_LOG: {
            if (n == 0u) {
                R_MAP1(log, TAPE(c, 0, op->a), r);
                return r;
            }
            /* (n b^[n] - sum_{j=1..n-1} j b^[n-j] a^[j]) / (n b0). */
            const real_t nb0 = R_SPLAT((double)n) * TAPE(c, 0, op->a);
            real_t ret = R_SPLAT((double)n) * TAPE(c, n, op->a);
            if (n > 1u) {
                ret = ret - conv(c, n, op->a, u_idx, 1, n - 1u, 1, zero);
            }
            return ret / nb0;
        }
        case HY_OP_TIME:
            return n == 0u ? time_v : (n == 1u ? R_SPLAT(1.) : zero);
        case HY_OP_CFUNC:
            return n == 0u ? cfunc_eval(c, op) : zero;
        case HY_OP_SIGMOID: {
            /* src/math/sigmoid.cpp:137-179 (default mode, pairwise) / :262-322 (compact mode, sequential):
             * (1/n) sum_{j=1..n} ((a^[n-j] - c^[n-j]) b^[j]) j, a = this u variable, c = a^2. */
            if (n == 0u) {
                R_MAP1(sigmoid_d, TAPE(c, 0, op->a), r);
                return r;
            }
            real_t buf[256];
            real_t acc = zero;
            for (uint32_t j = 1; j <= n; ++j) {
                const real_t t1 = TAPE(c, n - j, u_idx) - TAPE(c, n - j, op->c);
                const real_t t2 = t1 * TAPE(c, j, op->a);
                if (c->mode & ORACLE_PAIRWISE) {
                    buf[j - 1u] = t2 * R_SPLAT((double)j);
                } else {
                    acc = r_fma(c, R_SPLAT((double)j), t2, acc);
                }
            }
            if (c->mode & ORACLE_PAIRWISE) {
                acc = pairwise_sum(buf, n);
            }
            return acc / R_SPLAT((double)n);
        }
        case HY_OP_RELUP: {
            /* src/math/relu.cpp:404-424: relup(u^[0]) at order 0, zero afterwards. */
            if (n != 0u) {
                return zero;
            }
            const real_t x0 = TAPE(c, 0, op->a);
            for (int l_ = 0; l_ < ORACLE_W; ++l_) {
                R_SET(r, l_, R_GET(x0, l_) > 0. ? 1. : P->consts[op->b]);
            }
            return r;
        }
        case HY_OP_RELU: {
            /* src/math/relu.cpp:157-176: select(u^[0] > 0, u^[n], slope * u^[n]). */
            const real_t x0 = TAPE(c, 0, op->a), xn = TAPE(c, n, op->a);
            for (int l_ = 0; l_ < ORACLE_W; ++l_) {
                R_SET(r, l_, relu_d(R_GET(x0, l_), R_GET(xn, l_), P->consts[op->b]));
            }
            return r;
        }
    }
    return R_SPLAT(NAN);
}

/* State-variable derivative of order n >= 1 (src/taylor_02.cpp:245-287): true division by n. */
static real_t sv_diff(const ctx_t *c, uint32_t sv, uint32_t n)
{
    const uint32_t ref = c->P->sv_defs[sv];
    if (HY_REF_KIND(ref) == HY_REF_VAR) {
        return TAPE(c, n - 1u, HY_REF_IDX(ref)) / R_SPLAT((double)n);
    }
    return n == 1u ? numpar_val(c, ref) : R_SPLAT(0.);
}

#if ORACLE_W != 1
/* A generated (straight-line, per-order unrolled) jet for the program being run, see oracle/codegen.py: when
 * installed it replaces the interpreting loop below; the driver (step size, update, propagate loop) stays. The
 * caller guarantees that the installed function was generated for the program it then runs. */
typedef void (*jet_fn_t)(real_t *T, const real_t *par, const real_t *tm);
static jet_fn_t jet_hook = NULL;
void SYM(oracle_set_jet)(jet_fn_t f)
{
    jet_hook = f;
}
#endif

/* The whole jet: orders 0..p-1 for every u variable, order p for the state variables. */
static void compute_jet(ctx_t *c, const double *state, const double *t_hi)
{
    const hy_program_desc *P = c->P;
    real_t time_v = R_SPLAT(0.);

    for (uint32_t l = 0; l < ORACLE_W; ++l) {
        const uint32_t ll = l < c->nl ? l : c->nl - 1u;
        R_SET(time_v, l, t_hi[c->lane0 + ll]);
    }
    for (uint32_t i = 0; i < P->n_eq; ++i) {
        real_t v = R_SPLAT(0.);
#if ORACLE_W != 1
        if (c->nl == ORACLE_W) {
            memcpy(&v, state + (size_t)i * c->batch + c->lane0, sizeof(v)); /* the lanes of a variable are contiguous */
            TAPE(c, 0, i) = v;
            continue;
        }
#endif
        for (uint32_t l = 0; l < ORACLE_W; ++l) {
            const uint32_t ll = l < c->nl ? l : c->nl - 1u;
            R_SET(v, l, state[(size_t)i * c->batch + c->lane0 + ll]);
        }
        TAPE(c, 0, i) = v;
    }
#if ORACLE_W != 1
    if (jet_hook != NULL) {
        real_t parv[64];
        if (P->n_pars <= 64u) {
            for (uint32_t k = 0; k < P->n_pars; ++k) {
                parv[k] = load_par(c, k);
            }
            jet_hook(c->T, parv, &time_v);
            return;
        }
    }
#endif
    for (uint32_t n = 0; n < P->order; ++n) {
        if (n > 0u) {
            for (uint32_t i = 0; i < P->n_eq; ++i) {
                TAPE(c, n, i) = sv_diff(c, i, n);
            }
        }
        for (uint32_t i = P->n_eq; i < P->n_uvars; ++i) {
            TAPE(c, n, i) = diff_op(c, &P->ops[i - P->n_eq], i, n, time_v);
        }
    }
    for (uint32_t i = 0; i < P->n_eq; ++i) {
        TAPE(c, P->order, i) = sv_diff(c, i, P->order);
    }
}

/* ---- per-lane scalar tail: step size, state update ------------------------------------------ */

/* std::max / std::min semantics (src/detail/llvm_helpers_cmp.cpp:313-329). */
static inline double std_max(double a, double b)
{
    return (a < b) ? b : a;
}
static inline double std_min(double a, double b)
{
    return (b < a) ? b : a;
}

static double pairwise_max(double *v, uint32_t n)
{
    while (n != 1u) {
        uint32_t m = 0;
        for (uint32_t i = 0; i < n; i += 2u) {
            v[m++] = (i + 1u == n) ? v[i] : std_max(v[i], v[i + 1u]);
        }
        n = m;
    }
    return v[0];
}

/* taylor_determine_h_rhofac(), src/taylor_00.cpp:84-94. */
static double rhofac_of(uint32_t order)
{
    const double m7_10 = -7. / 10.;
    const double e2 = exp(1.) * exp(1.);
    return exp(m7_10 / (double)(order - 1u)) / e2;
}

/* taylor_determine_h(), src/taylor_00.cpp:102-273, for lane l of the group. */
static double determine_h(const ctx_t *c, uint32_t l, double max_delta_t)
{
    const hy_program_desc *P = c->P;
    const uint32_t p = P->order, n_eq = P->n_eq;
    double m0, mp, mp1;

    if (c->mode & ORACLE_PAIRWISE) {
        double *v0 = (double *)malloc(sizeof(double) * 3u * n_eq), *vp = v0 + n_eq, *vp1 = vp + n_eq;
        for (uint32_t i = 0; i < n_eq; ++i) {
            v0[i] = fabs(R_GET(TAPE(c, 0, i), l));
            vp[i] = fabs(R_GET(TAPE(c, p, i), l));
            vp1[i] = fabs(R_GET(TAPE(c, p - 1u, i), l));
        }
        m0 = pairwise_max(v0, n_eq);
        mp = pairwise_max(vp, n_eq);
        mp1 = pairwise_max(vp1, n_eq);
        free(v0);
    } else {
        m0 = fabs(R_GET(TAPE(c, 0, 0), l));
        mp = fabs(R_GET(TAPE(c, p, 0), l));
        mp1 = fabs(R_GET(TAPE(c, p - 1u, 0), l));
        for (uint32_t i = 1; i < n_eq; ++i) {
            m0 = std_max(m0, fabs(R_GET(TAPE(c, 0, i), l)));
            mp = std_max(mp, fabs(R_GET(TAPE(c, p, i), l)));
            mp1 = std_max(mp1, fabs(R_GET(TAPE(c, p - 1u, i), l)));
        }
    }

    const double num_rho = (m0 <= 1.) ? 1. : m0;
    const double rho_o = pow(num_rho / mp, 1. / (double)p);
    const double rho_om1 = pow(num_rho / mp1, 1. / (double)(p - 1u));
    const double rho_m = std_min(rho_o, rho_om1);
    double h = rho_m * rhofac_of(p);
    h = std_min(h, fabs(max_delta_t));
    return (max_delta_t < 0.) ? -1. * h : 1. * h;
}

/* taylor_run_multihorner() / taylor_run_ceval(), src/taylor_00.cpp:279-460, lane l. */
static void update_state(const ctx_t *c, uint32_t l, double h, double *state)
{
    const hy_program_desc *P = c->P;
    const uint32_t p = P->order, n_eq = P->n_eq;

    if (!P->high_accuracy) {
        for (uint32_t i = 0; i < n_eq; ++i) {
            double res = R_GET(TAPE(c, p, i), l);
            for (uint32_t o = 1; o <= p; ++o) {
#if ORACLE_W == 1
                res = (c->mode & ORACLE_FMA) ? fma(res, h, R_GET(TAPE(c, p - o, i), l))
                                             : R_GET(TAPE(c, p - o, i), l) + res * h;
#else
                res = R_GET(TAPE(c, p - o, i), l) + res * h;
#endif
            }
            state[(size_t)i * c->batch + c->lane0 + l] = res;
        }
    } else {
        for (uint32_t i = 0; i < n_eq; ++i) {
            double res = R_GET(TAPE(c, 0, i), l), comp = 0., cur_h = h;
            for (uint32_t o = 1; o <= p; ++o) {
                /* NOTE: the compensated sum must not be contracted or reassociated. */
                volatile double tmp = R_GET(TAPE(c, o, i), l) * cur_h;
                volatile double y = tmp - comp;
                volatile double t = res + y;
                volatile double d = t - res;
                comp = d - y;
                res = t;
                cur_h = cur_h * h;
            }
            state[(size_t)i * c->batch + c->lane0 + l] = res;
        }
    }
}

#if ORACLE_W != 1
/* ---- SIMD tail: the same step size and state update on all the lanes of the group at once -----
 * In the reference the step-size deduction and the state update are part of the JIT-compiled step function and
 * operate on SIMD vectors of batch_size lanes like the jet (src/taylor_00.cpp:102-460, :712-865). The timed CPU
 * baseline does the same; the operations of every lane are those of determine_h() / update_state() above, in the
 * same order (tests/test_codegen_cpu.py checks that the two tails agree to the bit). */
typedef long long imask_t __attribute__((vector_size(ORACLE_W * 8)));

static inline real_t v_abs(real_t x)
{
    const imask_t m = (imask_t){0} + 0x7fffffffffffffffll;
    return (real_t)((imask_t)x & m);
}
/* std::max(a, b) = (a < b) ? b : a, lane by lane. */
static inline real_t v_std_max(real_t a, real_t b)
{
    const imask_t m = a < b;
    return (real_t)(((imask_t)b & m) | ((imask_t)a & ~m));
}
static real_t v_pairwise_max(real_t *v, uint32_t n)
{
    while (n != 1u) {
        uint32_t m = 0;
        for (uint32_t i = 0; i < n; i += 2u) {
            v[m++] = (i + 1u == n) ? v[i] : v_std_max(v[i], v[i + 1u]);
        }
        n = m;
    }
    return v[0];
}

/* A value the optimiser cannot see through: keeps the product of the compensated summation from being fused
 * into the subtraction that follows it (-ffp-contract=fast is on in this build). Off the critical path. */
static inline real_t v_opaque(real_t x)
{
    __asm__("" : "+m"(x));
    return x;
}

static void step_tail_v(const ctx_t *c, double *state, double *h_inout)
{
    const hy_program_desc *P = c->P;
    const uint32_t p = P->order, n_eq = P->n_eq;
    real_t m0, mp, mp1, h;

    /* taylor_determine_h(): the three norms by SIMD maxima, the two pow() calls lane by lane. */
    if (c->mode & ORACLE_PAIRWISE) {
        real_t *v0 = c->T + (size_t)P->n_uvars * (p + 1u), *vp = v0 + n_eq, *vp1 = vp + n_eq;
        for (uint32_t i = 0; i < n_eq; ++i) {
            v0[i] = v_abs(TAPE(c, 0, i));
            vp[i] = v_abs(TAPE(c, p, i));
            vp1[i] = v_abs(TAPE(c, p - 1u, i));
        }
        m0 = v_pairwise_max(v0, n_eq);
        mp = v_pairwise_max(vp, n_eq);
        mp1 = v_pairwise_max(vp1, n_eq);
    } else {
        m0 = v_abs(TAPE(c, 0, 0));
        mp = v_abs(TAPE(c, p, 0));
        mp1 = v_abs(TAPE(c, p - 1u, 0));
        for (uint32_t i = 1; i < n_eq; ++i) {
            m0 = v_std_max(m0, v_abs(TAPE(c, 0, i)));
            mp = v_std_max(mp, v_abs(TAPE(c, p, i)));
            mp1 = v_std_max(mp1, v_abs(TAPE(c, p - 1u, i)));
        }
    }
    const double rhofac = rhofac_of(p);
    h = R_SPLAT(0.);
    for (uint32_t l = 0; l < ORACLE_W; ++l) {
        const uint32_t ll = l < c->nl ? l : c->nl - 1u;
        const double max_delta_t = h_inout[c->lane0 + ll];
        const double num_rho = (m0[l] <= 1.) ? 1. : m0[l];
        const double rho_o = pow(num_rho / mp[l], 1. / (double)p);
        const double rho_om1 = pow(num_rho / mp1[l], 1. / (double)(p - 1u));
        const double rho_m = std_min(rho_o, rho_om1);
        double hl = rho_m * rhofac;
        hl = std_min(hl, fabs(max_delta_t));
        h[l] = (max_delta_t < 0.) ? -1. * hl : 1. * hl;
    }

    /* taylor_run_multihorner() / taylor_run_ceval(). */
    for (uint32_t i = 0; i < n_eq; ++i) {
        real_t res;
        if (!P->high_accuracy) {
            res = TAPE(c, p, i);
            for (uint32_t o = 1; o <= p; ++o) {
                res = TAPE(c, p - o, i) + res * h;
            }
        } else {
            real_t comp = R_SPLAT(0.), cur_h = h;
            res = TAPE(c, 0, i);
            for (uint32_t o = 1; o <= p; ++o) {
                const real_t tmp = v_opaque(TAPE(c, o, i) * cur_h);
                const real_t y = tmp - comp;
                const real_t t = res + y;
                const real_t d = t - res;
                comp = d - y;
                res = t;
                cur_h = cur_h * h;
            }
        }
        double *dst = state + (size_t)i * c->batch + c->lane0;
        if (c->nl == ORACLE_W) {
            memcpy(dst, &res, sizeof(res));
        } else {
            for (uint32_t l = 0; l < c->nl; ++l) {
                dst[l] = res[l];
            }
        }
    }
    for (uint32_t l = 0; l < c->nl; ++l) {
        h_inout[c->lane0 + l] = h[l];
    }
}
#endif

/* ---- double-length time (include/heyoka/detail/dfloat.hpp:104-169) -------------------------- */
typedef struct {
    double hi, lo;
} dfl;

static inline dfl eft_knuth(double a, double b)
{
    volatile double x = a + b;
    volatile double z = x - a;
    volatile double y = (a - (x - z)) + (b - z);
    dfl r = {x, y};
    return r;
}
static inline dfl eft_dekker(double a, double b)
{
    volatile double x = a + b;
    volatile double y = (a - x) + b;
    dfl r = {x, y};
    return r;
}
static inline dfl dfl_add(dfl a, dfl b)
{
    const dfl h = eft_knuth(a.hi, b.hi);
    const dfl lo = eft_knuth(a.lo, b.lo);
    dfl uv = eft_dekker(h.hi, h.lo + lo.hi);
    uv = eft_dekker(uv.hi, uv.lo + lo.lo);
    return uv;
}
static inline dfl dfl_sub(dfl a, dfl b)
{
    const dfl nb = {-b.hi, -b.lo};
    return dfl_add(a, nb);
}
static inline int dfl_lt(dfl x, dfl y)
{
    return (x.hi < y.hi) || (x.hi == y.hi && x.lo < y.lo);
}
static inline int dfl_ge0(dfl x)
{
    /* x >= dfloat(0) */
    return (x.hi > 0.) || (x.hi == 0. && x.lo >= 0.);
}

/* ---- the JIT'd `step` function: jet + h + update (+ tc) for the lanes [lane0, lane0 + nl) ---- */
static void step_group(ctx_t *c, double *state, const double *t_hi, double *h_inout, double *tc)
{
    const hy_program_desc *P = c->P;

    compute_jet(c, state, t_hi);

#if ORACLE_W != 1
    if (!(c->mode & ORACLE_SCALAR_TAIL)) {
        step_tail_v(c, state, h_inout);
        if (tc != NULL) {
            for (uint32_t l = 0; l < c->nl; ++l) {
                for (uint32_t i = 0; i < P->n_eq; ++i) {
                    for (uint32_t o = 0; o <= P->order; ++o) {
                        tc[((size_t)i * (P->order + 1u) + o) * c->batch + c->lane0 + l] = R_GET(TAPE(c, o, i), l);
                    }
                }
            }
        }
        return;
    }
#endif
    for (uint32_t l = 0; l < c->nl; ++l) {
        const size_t lane = c->lane0 + l;
        const double h = determine_h(c, l, h_inout[lane]);
        update_state(c, l, h, state);
        h_inout[lane] = h;
        if (tc != NULL) {
            for (uint32_t i = 0; i < P->n_eq; ++i) {
                for (uint32_t o = 0; o <= P->order; ++o) {
                    tc[((size_t)i * (P->order + 1u) + o) * c->batch + lane] = R_GET(TAPE(c, o, i), l);
                }
            }
        }
    }
}

static real_t *alloc_tape(const hy_program_desc *P)
{
    void *p = NULL;
    const size_t n = (size_t)P->n_uvars * (P->order + 1u) + 3u * (size_t)P->n_eq; /* + scratch of the SIMD tail */
    if (posix_memalign(&p, 64, n * sizeof(real_t)) != 0) {
        return NULL;
    }
    return (real_t *)p;
}

/* Equivalent of the reference's step function pointer (include/heyoka/detail/ta_jit_data.hpp:35-38):
 * state RW, pars/time RO, h_inout in = signed max step, out = step taken, tc WO or NULL. */
int SYM(oracle_step)(const hy_program_desc *P, uint32_t batch, uint32_t lane_begin, uint32_t lane_end, double *state,
                     const double *pars, const double *t_hi, double *h_inout, double *tc, int mode)
{
    real_t *T = alloc_tape(P);
    if (T == NULL) {
        return 1;
    }
    for (uint32_t s = lane_begin; s < lane_end; s += ORACLE_W) {
        ctx_t c = {P, batch, s, 0, pars, T, mode};
        c.nl = lane_end - s < ORACLE_W ? lane_end - s : ORACLE_W;
        step_group(&c, state, t_hi, h_inout, tc);
    }
    free(T);
    return 0;
}

/* step_impl() (src/taylor_adaptive_batch.cpp:632-727): the step plus time update and outcome. */
int SYM(oracle_step_full)(const hy_program_desc *P, uint32_t batch, uint32_t lane_begin, uint32_t lane_end,
                          double *state, const double *pars, double *t_hi, double *t_lo, const double *max_delta_t,
                          double *last_h, int64_t *outcome, double *tc, int mode)
{
    double *h = (double *)malloc(sizeof(double) * batch);
    if (h == NULL) {
        return 1;
    }
    memcpy(h, max_delta_t, sizeof(double) * batch);
    const int err = SYM(oracle_step)(P, batch, lane_begin, lane_end, state, pars, t_hi, h, tc, mode);
    for (uint32_t i = lane_begin; i < lane_end && !err; ++i) {
        const dfl t = {t_hi[i], t_lo[i]}, hh = {h[i], 0.};
        const dfl nt = dfl_add(t, hh);
        t_hi[i] = nt.hi;
        t_lo[i] = nt.lo;
        last_h[i] = h[i];
        int nf = !(isfinite(nt.hi) && isfinite(nt.lo));
        for (uint32_t v = 0; v < P->n_eq && !nf; ++v) {
            nf = !isfinite(state[(size_t)v * batch + i]);
        }
        outcome[i] = nf ? HY_OUTCOME_ERR_NF_STATE : (h[i] == max_delta_t[i] ? HY_OUTCOME_TIME_LIMIT : HY_OUTCOME_SUCCESS);
    }
    free(h);
    return err;
}

/* propagate_until_impl() (src/taylor_adaptive_batch.cpp:1136-1534) restricted to what the hot path
 * supports: no callback, no continuous output. Lanes are independent, so each group of ORACLE_W lanes
 * iterates on its own; the *global* exits of the reference (any lane non-finite -> everybody stops
 * at that iteration; iteration limit) are reproduced exactly by tracking the iteration index:
 * `lockstep` != 0 runs the lanes [lane_begin, lane_end) in lock step like the reference (used by the
 * parity tests), `lockstep` == 0 lets every group of ORACLE_W lanes run to completion on its own (used
 * by the timed CPU baseline, where the global exits never fire). Threading is done by the caller:
 * disjoint lane ranges may be processed concurrently (no shared mutable state). */
int SYM(oracle_propagate_until)(const hy_program_desc *P, uint32_t batch, uint32_t lane_begin, uint32_t lane_end,
                                double *state, const double *pars, double *t_hi, double *t_lo, const double *tf_hi,
                                const double *tf_lo, const double *max_delta_t, uint64_t max_steps, double *last_h,
                                int64_t *outcome, double *min_h, double *max_h, uint64_t *n_steps, double *tc, int mode,
                                int lockstep)
{
    const uint32_t n_lanes = lane_end - lane_begin;
    const uint32_t n_groups = lockstep ? 1u : (n_lanes + ORACLE_W - 1u) / ORACLE_W;
    int err = 0;

    for (uint32_t i = lane_begin; i < lane_end; ++i) {
        n_steps[i] = 0;
        min_h[i] = INFINITY;
        max_h[i] = 0.;
    }

    {
        real_t *T = alloc_tape(P);
        double *cur = (double *)malloc(sizeof(double) * batch * 4u);
        if (T == NULL || cur == NULL) {
            err = 1;
        } else {
            double *cur_max = cur, *rem_hi = cur + batch, *rem_lo = rem_hi + batch, *hbuf = rem_lo + batch;
            for (uint32_t g = 0; g < n_groups; ++g) {
                const uint32_t l0 = lockstep ? lane_begin : lane_begin + g * ORACLE_W;
                const uint32_t l1 = lockstep ? lane_end : (l0 + ORACLE_W < lane_end ? l0 + ORACLE_W : lane_end);
                uint64_t iter = 0;

                for (uint32_t i = l0; i < l1; ++i) {
                    const dfl tf = {tf_hi[i], tf_lo ? tf_lo[i] : 0.}, t = {t_hi[i], t_lo[i]};
                    const dfl rem = dfl_sub(tf, t);
                    rem_hi[i] = rem.hi;
                    rem_lo[i] = rem.lo;
                }

                for (;;) {
                    /* direction is fixed by the initial remaining time; rem == 0 afterwards is either. */
                    for (uint32_t i = l0; i < l1; ++i) {
                        const dfl rem = {rem_hi[i], rem_lo[i]};
                        const double mdt = max_delta_t ? max_delta_t[i] : INFINITY;
                        const dfl lim_p = {mdt, 0.}, lim_m = {-mdt, 0.};
                        /* t_dir = rem >= 0 (computed once in the reference; rem never changes sign). */
                        const int dir = dfl_ge0(rem);
                        const dfl dt = dir ? (dfl_lt(rem, lim_p) ? rem : lim_p) : (dfl_lt(rem, lim_m) ? lim_m : rem);
                        cur_max[i] = dt.hi;
                        hbuf[i] = dt.hi;
                    }

                    /* One step for the lanes of this group. */
                    for (uint32_t s = l0; s < l1; s += ORACLE_W) {
                        ctx_t c = {P, batch, s, 0, pars, T, mode};
                        c.nl = l1 - s < ORACLE_W ? l1 - s : ORACLE_W;
                        step_group(&c, state, t_hi, hbuf, tc);
                    }

                    uint32_t n_done = 0;
                    int nf_any = 0;
                    for (uint32_t i = l0; i < l1; ++i) {
                        const double h = hbuf[i];
                        const dfl t = {t_hi[i], t_lo[i]}, hh = {h, 0.};
                        const dfl nt = dfl_add(t, hh);
                        t_hi[i] = nt.hi;
                        t_lo[i] = nt.lo;
                        last_h[i] = h;
                        int nf = !(isfinite(nt.hi) && isfinite(nt.lo));
                        for (uint32_t v = 0; v < P->n_eq && !nf; ++v) {
                            nf = !isfinite(state[(size_t)v * batch + i]);
                        }
                        if (nf) {
                            outcome[i] = HY_OUTCOME_ERR_NF_STATE;
                            nf_any = 1;
                            continue;
                        }
                        const int64_t oc = (h == cur_max[i]) ? HY_OUTCOME_TIME_LIMIT : HY_OUTCOME_SUCCESS;
                        n_steps[i] += (h != 0.);
                        if (oc == HY_OUTCOME_SUCCESS) {
                            const double ah = fabs(h);
                            min_h[i] = ah < min_h[i] ? ah : min_h[i];
                            max_h[i] = max_h[i] < ah ? ah : max_h[i];
                        }
                        const int done = (h == rem_hi[i]);
                        n_done += (uint32_t)done;
                        if (done) {
                            rem_hi[i] = 0.;
                            rem_lo[i] = 0.;
                        } else {
                            const dfl tf = {tf_hi[i], tf_lo ? tf_lo[i] : 0.};
                            const dfl rem = dfl_sub(tf, nt);
                            rem_hi[i] = rem.hi;
                            rem_lo[i] = rem.lo;
                        }
                        outcome[i] = oc;
                    }
                    if (nf_any) {
                        break;
                    }
                    ++iter;
                    if (n_done == l1 - l0) {
                        break;
                    }
                    if (iter == max_steps) {
                        for (uint32_t i = l0; i < l1; ++i) {
                            outcome[i] = HY_OUTCOME_STEP_LIMIT;
                        }
                        break;
                    }
                }
            }
        }
        free(T);
        free(cur);
    }
    return err;
}

/* Dense output (src/taylor_01.cpp:1015-1185): out[var][lane] = sum_o tc[var][o][lane] tau^o, by Horner
 * (or compensated summation in high-accuracy mode). */
int SYM(oracle_d_output)(const hy_program_desc *P, uint32_t batch, const double *tc, const double *tau, double *out)
{
    const uint32_t p = P->order;
    for (uint32_t i = 0; i < P->n_eq; ++i) {
        for (uint32_t l = 0; l < batch; ++l) {
            const double h = tau[l];
            const double *cf = tc + (size_t)i * (p + 1u) * batch + l;
            if (!P->high_accuracy) {
                double res = cf[(size_t)p * batch];
                for (uint32_t o = 1; o <= p; ++o) {
                    res = cf[(size_t)(p - o) * batch] + res * h;
                }
                out[(size_t)i * batch + l] = res;
            } else {
                double res = cf[0], comp = 0., cur_h = h;
                for (uint32_t o = 1; o <= p; ++o) {
                    volatile double tmp = cf[(size_t)o * batch] * cur_h;
                    volatile double y = tmp - comp;
                    volatile double t = res + y;
                    volatile double d = t - res;
                    comp = d - y;
                    res = t;
                    cur_h = cur_h * h;
                }
                out[(size_t)i * batch + l] = res;
            }
        }
    }
    return 0;
}

/* ================================================================================================
 * Event detection in batch mode (scalar build only): restatement of
 *   src/taylor_00.cpp:593-710           taylor_add_adaptive_step_with_events(): jet of the state variables AND of the
 *                                       event equations, step size from both, no propagation of the state;
 *   src/taylor_adaptive_batch.cpp:728-1035  the events branch of step_impl();
 *   src/detail/event_detection.cpp:1733-2173  ed_data_batch<T>::detect_events() with its helpers (:171-280 polynomial
 *                                       utilities, :413-507 translation by 1, :598-697 reverse-translate-count,
 *                                       :704-816 fast exclusion check, :519-550 automatic cooldown);
 *   src/detail/llvm_helpers_ed.cpp:58-330  sign-change count, interval enclosure by Horner.
 * The bracketed root finder is boost::math::tools::toms748_solve (Boost.Math, a dependency that is NOT in
 * /root/reference; heyoka requires Boost >= 1.69, no pinned version): Algorithm 748 of Alefeld, Potra and Shi (ACM TOMS
 * 21(3), 1995) restated below from the published algorithm in the arrangement Boost uses (secant, quadratic, two
 * cubic/quadratic steps, double-length secant, optional bisection per iteration; eps_tolerance = 4 eps). Event times
 * are therefore pinned to the reference by tolerance (its own tests use 1000 eps, test/batch_event_detection.cpp:158),
 * not bit for bit.
 * ============================================================================================== */
#if ORACLE_W == 1

#include <errno.h>
#include <float.h>

typedef struct {
    uint32_t lane;    /* batch index */
    uint32_t idx;     /* index among the terminal (terminal != 0) or non-terminal events */
    int32_t terminal;
    int32_t d_sgn;    /* sign of the time derivative of the event equation at the root */
    double t;         /* time of the event relative to the beginning of the step */
    double abs_der;
} oracle_event;

static inline int sgn_d(double x)
{
    return (0. < x) - (x < 0.);
}

/* :269-280 */
static double ed_poly_eval(const double *a, double x, uint32_t n)
{
    double ret = a[n];
    for (uint32_t i = 1; i <= n; ++i) {
        ret = a[n - i] + ret * x;
    }
    return ret;
}

/* :249-264 */
static double ed_poly_eval_1(const double *a, double x, uint32_t n)
{
    double ret1 = a[n] * (double)n;
    for (uint32_t i = 1; i < n; ++i) {
        ret1 = a[n - i] * (double)(n - i) + ret1 * x;
    }
    return ret1;
}

/* :171-192 */
static void ed_poly_rescale(double *ret, const double *a, double scal, uint32_t n)
{
    double cur_f = 1.;
    for (uint32_t i = 0; i <= n; ++i) {
        ret[i] = a[i] * cur_f;
        cur_f *= scal;
    }
}

/* :197-221 */
static void ed_poly_rescale_p2(double *ret, const double *a, uint32_t n)
{
    double cur_f = 1.;
    for (uint32_t i = 0; i <= n; ++i) {
        ret[n - i] = cur_f * a[n - i];
        cur_f *= 2.;
    }
}

/* :413-507 with the binomial table of llvm_helpers_ed.cpp:421-455. */
static void ed_poly_translate_1(double *out, const double *a, uint32_t n, const double *bc)
{
    for (uint32_t i = 0; i <= n; ++i) {
        out[i] = 0.;
    }
    for (uint32_t i = 0; i <= n; ++i) {
        for (uint32_t k = 0; k <= i; ++k) {
            out[k] = out[k] + a[i] * bc[i * (n + 1u) + k];
        }
    }
}

/* llvm_helpers_ed.cpp:58-190: number of sign changes, zeros skipped. */
static uint32_t ed_count_sign_changes(const double *a, uint32_t n)
{
    uint32_t last_nz = 0, ret = 0;
    for (uint32_t i = 1; i <= n; ++i) {
        const int cur = sgn_d(a[i]), last = sgn_d(a[last_nz]);
        ret += (last != 0 && cur + last == 0) ? 1u : 0u;
        if (cur != 0) {
            last_nz = i;
        }
    }
    return ret;
}

/* :598-697: reverse a into t1, translate by 1 into t2, count the sign changes of t2. */
static uint32_t ed_rtscc(double *t1, double *t2, const double *a, uint32_t n, const double *bc)
{
    for (uint32_t i = 0; i <= n; ++i) {
        t1[i] = a[n - i];
    }
    ed_poly_translate_1(t2, t1, n, bc);
    return ed_count_sign_changes(t2, n);
}

/* :704-816 (use_cs == false) + llvm_helpers_ed.cpp:227-330: enclosure of the polynomial over [0, h] (or [h, 0]) by
 * Horner's scheme in interval arithmetic; true = no sign change possible. */
static int ed_fex_check(const double *a, uint32_t n, double h, int back)
{
    const double h_lo = back ? h : 0., h_hi = back ? 0. : h;
    double acc_lo = a[n], acc_hi = a[n];
    for (uint32_t i = 1; i <= n; ++i) {
        const double cf = a[n - i];
        const double t1 = acc_lo * h_lo, t2 = acc_lo * h_hi, t3 = acc_hi * h_lo, t4 = acc_hi * h_hi;
        const double lo = std_min(std_min(t1, t2), std_min(t3, t4));
        const double hi = std_max(std_max(t1, t2), std_max(t3, t4));
        acc_lo = cf + lo;
        acc_hi = cf + hi;
    }
    const int s_lo = sgn_d(acc_lo), s_hi = sgn_d(acc_hi);
    return s_lo == s_hi && s_lo != 0;
}

/* ---- TOMS 748 (see the header of this section) ---- */
typedef struct {
    const double *poly;
    uint32_t order;
} t748_f;

static inline double t748_eval(const t748_f *f, double x)
{
    return ed_poly_eval(f->poly, x, f->order);
}
static inline int t748_sign(double z)
{
    return z == 0. ? 0 : (signbit(z) ? -1 : 1);
}
static inline int t748_tol(double a, double b)
{
    return fabs(a - b) <= 4. * DBL_EPSILON * fmin(fabs(a), fabs(b));
}
static inline double t748_safe_div(double num, double denom, double r)
{
    if (fabs(denom) < 1.) {
        if (fabs(denom * DBL_MAX) <= fabs(num)) {
            return r;
        }
    }
    return num / denom;
}
static void t748_bracket(const t748_f *f, double *a, double *b, double c, double *fa, double *fb, double *d, double *fd)
{
    const double tol = DBL_EPSILON * 2.;
    if ((*b - *a) < 2. * tol * *a) {
        c = *a + (*b - *a) / 2.;
    } else if (c <= *a + fabs(*a) * tol) {
        c = *a + fabs(*a) * tol;
    } else if (c >= *b - fabs(*b) * tol) {
        c = *b - fabs(*b) * tol;
    }
    const double fc = t748_eval(f, c);
    if (fc == 0.) {
        *a = c;
        *fa = 0.;
        *d = 0.;
        *fd = 0.;
        return;
    }
    if (t748_sign(*fa) * t748_sign(fc) < 0) {
        *d = *b;
        *fd = *fb;
        *b = c;
        *fb = fc;
    } else {
        *d = *a;
        *fd = *fa;
        *a = c;
        *fa = fc;
    }
}
static double t748_secant(double a, double b, double fa, double fb)
{
    const double tol = DBL_EPSILON * 5.;
    const double c = a - (fa / (fb - fa)) * (b - a);
    if (c <= a + fabs(a) * tol || c >= b - fabs(b) * tol) {
        return (a + b) / 2.;
    }
    return c;
}
static double t748_quadratic(double a, double b, double d, double fa, double fb, double fd, unsigned count)
{
    double B = t748_safe_div(fb - fa, b - a, DBL_MAX);
    double A = t748_safe_div(fd - fb, d - b, DBL_MAX);
    A = t748_safe_div(A - B, d - a, 0.);
    if (A == 0.) {
        return t748_secant(a, b, fa, fb);
    }
    double c = (t748_sign(A) * t748_sign(fa) > 0) ? a : b;
    for (unsigned i = 1; i <= count; ++i) {
        c -= t748_safe_div(fa + (B + A * (c - b)) * (c - a), B + A * (2. * c - a - b), 1. + c - a);
    }
    if (c <= a || c >= b) {
        c = t748_secant(a, b, fa, fb);
    }
    return c;
}
static double t748_cubic(double a, double b, double d, double e, double fa, double fb, double fd, double fe)
{
    const double q11 = (d - e) * fd / (fe - fd);
    const double q21 = (b - d) * fb / (fd - fb);
    const double q31 = (a - b) * fa / (fb - fa);
    const double d21 = (b - d) * fd / (fd - fb);
    const double d31 = (a - b) * fb / (fb - fa);
    const double q22 = (d21 - q11) * fb / (fe - fb);
    const double q32 = (d31 - q21) * fa / (fd - fa);
    const double d32 = (d31 - q21) * fd / (fd - fa);
    const double q33 = (d32 - q22) * fa / (fe - fa);
    double c = q31 + q32 + q33 + a;
    if (c <= a || c >= b) {
        c = t748_quadratic(a, b, d, fa, fb, fd, 3);
    }
    return c;
}
static inline int t748_prof(double fa, double fb, double fd, double fe)
{
    const double m = DBL_MIN * 32.;
    return fabs(fa - fb) < m || fabs(fa - fd) < m || fabs(fa - fe) < m || fabs(fb - fd) < m || fabs(fb - fe) < m
           || fabs(fd - fe) < m;
}
/* Returns the bracket [*ra, *rb]; *max_iter in: limit, out: evaluations used; *err = EDOM if [ax, bx] is not a bracket. */
static void t748_solve(const t748_f *f, double ax, double bx, uint64_t *max_iter, double *ra, double *rb, int *err)
{
    *err = 0;
    if (*max_iter <= 2u) {
        *ra = ax;
        *rb = bx;
        return;
    }
    *max_iter -= 2u;
    uint64_t count = *max_iter;
    double a = ax, b = bx, fa = t748_eval(f, ax), fb = t748_eval(f, bx), c, u, fu, a0, b0, d, fd, e, fe;
    const double mu = 0.5;
    if (a >= b) {
        *err = EDOM;
        *ra = *rb = NAN;
        *max_iter += 2u;
        return;
    }
    if (t748_tol(a, b) || fa == 0. || fb == 0.) {
        *max_iter = 0;
        if (fa == 0.) {
            b = a;
        } else if (fb == 0.) {
            a = b;
        }
        *ra = a;
        *rb = b;
        *max_iter += 2u;
        return;
    }
    if (t748_sign(fa) * t748_sign(fb) > 0) {
        *err = EDOM;
        *ra = *rb = NAN;
        *max_iter += 2u;
        return;
    }
    fe = e = fd = 1e5;
    d = 0.;
    if (fa != 0.) {
        c = t748_secant(a, b, fa, fb);
        t748_bracket(f, &a, &b, c, &fa, &fb, &d, &fd);
        --count;
        if (count && fa != 0. && !t748_tol(a, b)) {
            c = t748_quadratic(a, b, d, fa, fb, fd, 2);
            e = d;
            fe = fd;
            t748_bracket(f, &a, &b, c, &fa, &fb, &d, &fd);
            --count;
        }
    }
    while (count && fa != 0. && !t748_tol(a, b)) {
        a0 = a;
        b0 = b;
        if (t748_prof(fa, fb, fd, fe)) {
            c = t748_quadratic(a, b, d, fa, fb, fd, 2);
        } else {
            c = t748_cubic(a, b, d, e, fa, fb, fd, fe);
        }
        e = d;
        fe = fd;
        t748_bracket(f, &a, &b, c, &fa, &fb, &d, &fd);
        if (0u == --count || fa == 0. || t748_tol(a, b)) {
            break;
        }
        if (t748_prof(fa, fb, fd, fe)) {
            c = t748_quadratic(a, b, d, fa, fb, fd, 3);
        } else {
            c = t748_cubic(a, b, d, e, fa, fb, fd, fe);
        }
        t748_bracket(f, &a, &b, c, &fa, &fb, &d, &fd);
        if (0u == --count || fa == 0. || t748_tol(a, b)) {
            break;
        }
        if (fabs(fa) < fabs(fb)) {
            u = a;
            fu = fa;
        } else {
            u = b;
            fu = fb;
        }
        c = u - 2. * (fu / (fb - fa)) * (b - a);
        if (fabs(c - u) > (b - a) / 2.) {
            c = a + (b - a) / 2.;
        }
        e = d;
        fe = fd;
        t748_bracket(f, &a, &b, c, &fa, &fb, &d, &fd);
        if (0u == --count || fa == 0. || t748_tol(a, b)) {
            break;
        }
        if ((b - a) < mu * (b0 - a0)) {
            continue;
        }
        e = d;
        fe = fd;
        t748_bracket(f, &a, &b, a + (b - a) / 2., &fa, &fb, &d, &fd);
        --count;
    }
    *max_iter -= count;
    if (fa == 0.) {
        b = a;
    } else if (fb == 0.) {
        a = b;
    }
    *ra = a;
    *rb = b;
    *max_iter += 2u;
}

/* :307-394: the only root of poly in [lb, ub). cflag: 0 ok, -1 too many iterations, > 0 errno. */
static double ed_bracketed_root_find(const double *poly, uint32_t order, double lb, double ub, int *cflag)
{
    if (isfinite(lb) && isfinite(ub) && ub > lb) {
        ub = nextafter(ub, lb);
    }
    const uint64_t iter_limit = DBL_MANT_DIG;
    uint64_t max_iter = iter_limit;
    const t748_f f = {poly, order};
    double a, b;
    int err;
    t748_solve(&f, lb, ub, &max_iter, &a, &b, &err);
    const double ret = a / 2. + b / 2.;
    if (err > 0) {
        *cflag = err;
        return 0.;
    }
    *cflag = max_iter < iter_limit ? 0 : -1;
    return ret;
}

/* :519-550 */
static double ed_deduce_cooldown(double g_eps, double abs_der)
{
    const double ret = g_eps / abs_der * 10.;
    return isfinite(ret) ? ret : 0.;
}

typedef struct {
    oracle_event *v;
    uint32_t n, cap;
} ev_list;

static void ev_push(ev_list *L, oracle_event e)
{
    if (L->n == L->cap) {
        L->cap = L->cap ? 2u * L->cap : 16u;
        L->v = (oracle_event *)realloc(L->v, sizeof(oracle_event) * L->cap);
    }
    L->v[L->n++] = e;
}

/* add_d_event (:1841-1912): the root is already rescaled to [0, h). */
static void ed_add_d_event(const double *ptr, uint32_t order, double h, int dir, oracle_event proto, ev_list *out,
                           double root)
{
    if (!isfinite(root)) {
        return;
    }
    if (fabs(root) >= fabs(h)) {
        root = nextafter(h, 0.);
    }
    const double der = ed_poly_eval_1(ptr, root, order);
    if (!isfinite(der)) {
        return;
    }
    const int d_sgn = sgn_d(der);
    if (dir == 0 || d_sgn == dir) {
        proto.t = root;
        proto.d_sgn = d_sgn;
        proto.abs_der = fabs(der);
        ev_push(out, proto);
    }
}

/* Deepest working list of the root isolation since the last oracle_ev_max_depth_w1(1) call. A readout for the tests: the
 * device keeps this list in a fixed stack of EV_STACK entries (ev_kernels.cuh), the reference in a list it gives up on
 * past 250 entries. Not read by anything else. */
static uint32_t ed_max_wl = 0u;

uint32_t oracle_ev_max_depth_w1(int reset)
{
    const uint32_t ret = ed_max_wl;
    if (reset) {
        ed_max_wl = 0u;
    }
    return ret;
}

/* The body of run_detection() (:1767-2168) for one batch element and one event: the polynomial of the event is
 * ptr[0..order], dir the requested direction, cd = {time in cooldown, cooldown} or NULL. */
static void ed_detect_one(const double *ptr, uint32_t order, double h, double g_eps, int dir, const double *cd,
                          const double *bc, oracle_event proto, ev_list *out)
{
    if (!isfinite(h) || !isfinite(g_eps) || h == 0.) {
        return;
    }
    const uint32_t np1 = order + 1u;
    double *isol = (double *)malloc(sizeof(double) * 2u * (order + 2u));
    uint32_t n_isol = 0;
    /* Working list: (lb, ub, polynomial). */
    const uint32_t wl_cap = 256u;
    double *wl_b = (double *)malloc(sizeof(double) * 2u * wl_cap);
    double *wl_p = (double *)malloc(sizeof(double) * (size_t)np1 * wl_cap);
    double *tmp = (double *)malloc(sizeof(double) * 3u * np1), *tmp1 = tmp + np1, *tmp2 = tmp1 + np1;
    uint32_t n_wl = 0;


    double lb_offset = 0.;
    if (cd != NULL) {
        lb_offset = (h >= 0.) ? (cd[1] - cd[0]) / fabs(h) : (cd[1] + cd[0]) / fabs(h);
    }
    if (lb_offset >= 1.) {
        goto done;
    }
    ed_poly_rescale(tmp, ptr, h, order);
    wl_b[0] = 0.;
    wl_b[1] = 1.;
    memcpy(wl_p, tmp, sizeof(double) * np1);
    n_wl = 1;
    int loop_failed = 0;
    do {
        const double lb = wl_b[2u * (n_wl - 1u)], ub = wl_b[2u * (n_wl - 1u) + 1u];
        memcpy(tmp, wl_p + (size_t)(n_wl - 1u) * np1, sizeof(double) * np1);
        --n_wl;
        int all_fin = 1;
        for (uint32_t k = 1; k <= order; ++k) {
            all_fin = all_fin && isfinite(tmp[k]);
        }
        if (tmp[0] == 0. && all_fin) {
            const int skip_event = cd != NULL && lb < lb_offset;
            if (!skip_event) {
                ed_add_d_event(ptr, order, h, dir, proto, out, lb * h);
            }
        }
        const uint32_t n_sc = ed_rtscc(tmp1, tmp2, tmp, order, bc);
        if (n_sc == 1u) {
            isol[2u * n_isol] = lb;
            isol[2u * n_isol + 1u] = ub;
            ++n_isol;
        } else if (n_sc > 1u) {
            ed_poly_rescale_p2(tmp1, tmp, order);
            ed_poly_translate_1(tmp2, tmp1, order, bc);
            const double mid = lb / 2. + ub / 2.;
            if (lb_offset < mid) {
                wl_b[2u * n_wl] = lb;
                wl_b[2u * n_wl + 1u] = mid;
                memcpy(wl_p + (size_t)n_wl * np1, tmp1, sizeof(double) * np1);
                ++n_wl;
            }
            wl_b[2u * n_wl] = mid;
            wl_b[2u * n_wl + 1u] = ub;
            memcpy(wl_p + (size_t)n_wl * np1, tmp2, sizeof(double) * np1);
            ++n_wl;
            ed_max_wl = n_wl > ed_max_wl ? n_wl : ed_max_wl;
        }
        if (n_wl > 250u || n_isol > order) {
            loop_failed = 1;
            break;
        }
    } while (n_wl != 0u);
    if (n_isol == 0u || loop_failed) {
        goto done;
    }
    ed_poly_rescale(tmp1, ptr, h, order);
    for (uint32_t k = 0; k < n_isol; ++k) {
        double lb = isol[2u * k];
        const double ub = isol[2u * k + 1u];
        if (cd != NULL && lb < lb_offset) {
            lb = lb_offset;
            const double f_lb = ed_poly_eval(tmp1, lb, order), f_ub = ed_poly_eval(tmp1, ub, order);
            if (!(f_lb * f_ub < 0.)) {
                continue;
            }
        }
        int cflag;
        const double root = ed_bracketed_root_find(tmp1, order, lb, ub, &cflag);
        if (cflag == 0) {
            ed_add_d_event(ptr, order, h, dir, proto, out, root * h);
        }
    }
done:
    free(isol);
    free(wl_b);
    free(wl_p);
    free(tmp);
}

static int ev_cmp_abs_t(const void *a, const void *b)
{
    const double x = fabs(((const oracle_event *)a)->t), y = fabs(((const oracle_event *)b)->t);
    return (x < y) ? -1 : (y < x ? 1 : 0);
}

/* One step of a batch integrator with events (the events branch of step_impl()). P->n_ev event equations, the first
 * n_te of them terminal; dirs[n_ev] in {-1, 0, 1}; cooldowns[n_te] (< 0: automatic); cd[batch][n_te][2] and
 * cd_on[batch][n_te] the cooldown state ({time spent, cooldown}, active flag), updated in place;
 * tc[(n_eq + n_ev)][p + 1][batch] written unconditionally (:776). Events out: for every lane (ascending) the
 * non-terminal events that happen before the first terminal one, in time order, then the first terminal event if
 * any. outcome[lane] = -idx - 1 for a terminal event (the caller turns it into idx if its callback returns true).
 * Callbacks and their exceptions are the caller's business. */
int oracle_step_ev_w1(const hy_program_desc *P, uint32_t batch, double *state, const double *pars, double *t_hi,
                      double *t_lo, const double *max_delta_t, double tol, uint32_t n_te, const int32_t *dirs,
                      const double *cooldowns, double *cd, int32_t *cd_on, double *tc, double *last_h, int64_t *outcome,
                      oracle_event *evs, uint32_t evs_cap, uint32_t *n_evs, int mode)
{
    const uint32_t p = P->order, n_eq = P->n_eq, n_ev = P->n_ev, pp1 = p + 1u;
    real_t *T = alloc_tape(P);
    double *bc = (double *)malloc(sizeof(double) * pp1 * pp1), *poly = (double *)malloc(sizeof(double) * pp1);
    if (T == NULL || bc == NULL || poly == NULL) {
        return 1;
    }
    /* Binomial coefficients (exact in double for the orders in use). */
    for (uint32_t i = 0; i <= p; ++i) {
        for (uint32_t j = 0; j <= p; ++j) {
            bc[i * pp1 + j] = j > i ? 0. : (j == 0u ? 1. : bc[(i - 1u) * pp1 + j - 1u] + (j <= i - 1u ? bc[(i - 1u) * pp1 + j] : 0.));
        }
    }
    uint32_t max_svf = 0;
    for (uint32_t k = 0; k < n_ev; ++k) {
        max_svf = P->ev_defs[k] > max_svf ? P->ev_defs[k] : max_svf;
    }
    *n_evs = 0;
    int overflow = 0;
    for (uint32_t lane = 0; lane < batch; ++lane) {
        ctx_t c = {P, batch, lane, 1, pars, T, mode};
        /* ---- jet (src/taylor_02.cpp:1211-1330 with sv_funcs: order p of the u variables up to max_svf_idx) ---- */
        compute_jet(&c, state, t_hi);
        if (max_svf >= n_eq) {
            const real_t time_v = t_hi[lane];
            for (uint32_t i = n_eq; i <= max_svf; ++i) {
                TAPE(&c, p, i) = diff_op(&c, &P->ops[i - n_eq], i, p, time_v);
            }
        }
        /* ---- step size (src/taylor_00.cpp:102-273, the sv_funcs take part in the three norms) ---- */
        const double mdt = max_delta_t != NULL ? max_delta_t[lane] : INFINITY;
        double m0, mp, mp1;
        {
            const uint32_t nn = n_eq + n_ev;
            double *v0 = (double *)malloc(sizeof(double) * 3u * nn), *vp = v0 + nn, *vp1 = vp + nn;
            for (uint32_t i = 0; i < nn; ++i) {
                const uint32_t u = i < n_eq ? i : P->ev_defs[i - n_eq];
                v0[i] = fabs(TAPE(&c, 0, u));
                vp[i] = fabs(TAPE(&c, p, u));
                vp1[i] = fabs(TAPE(&c, p - 1u, u));
            }
            if (mode & ORACLE_PAIRWISE) {
                m0 = pairwise_max(v0, nn);
                mp = pairwise_max(vp, nn);
                mp1 = pairwise_max(vp1, nn);
            } else {
                m0 = v0[0];
                mp = vp[0];
                mp1 = vp1[0];
                for (uint32_t i = 1; i < nn; ++i) {
                    m0 = std_max(m0, v0[i]);
                    mp = std_max(mp, vp[i]);
                    mp1 = std_max(mp1, vp1[i]);
                }
            }
            free(v0);
        }
        const double num_rho = (m0 <= 1.) ? 1. : m0;
        const double rho_m = std_min(pow(num_rho / mp, 1. / (double)p), pow(num_rho / mp1, 1. / (double)(p - 1u)));
        double h = std_min(rho_m * rhofac_of(p), fabs(mdt));
        h = (mdt < 0.) ? -1. * h : 1. * h;
        /* ---- g_eps (src/taylor_adaptive_batch.cpp:746-773) ---- */
        double g_eps;
        if (isfinite(m0)) {
            const double max_r_size = m0 < 1. ? tol : tol * m0;
            g_eps = max_r_size < DBL_EPSILON * m0 ? DBL_EPSILON * m0 : max_r_size;
        } else {
            g_eps = INFINITY;
        }
        /* ---- Taylor coefficients of the state variables and of the event equations ---- */
        for (uint32_t i = 0; i < n_eq + n_ev; ++i) {
            const uint32_t u = i < n_eq ? i : P->ev_defs[i - n_eq];
            for (uint32_t o = 0; o <= p; ++o) {
                tc[((size_t)i * pp1 + o) * batch + lane] = TAPE(&c, o, u);
            }
        }
        /* ---- detection ---- */
        ev_list d_tes = {NULL, 0, 0}, d_ntes = {NULL, 0, 0};
        for (uint32_t k = 0; k < n_ev; ++k) {
            for (uint32_t o = 0; o <= p; ++o) {
                poly[o] = tc[((size_t)(n_eq + k) * pp1 + o) * batch + lane];
            }
            if (ed_fex_check(poly, p, h, h < 0.)) {
                continue;
            }
            const int term = k < n_te;
            const oracle_event proto = {lane, term ? k : k - n_te, term, 0, 0., 0.};
            const double *cdp = (term && cd_on[(size_t)lane * n_te + k]) ? cd + ((size_t)lane * n_te + k) * 2u : NULL;
            ed_detect_one(poly, p, h, g_eps, dirs[k], cdp, bc, proto, term ? &d_tes : &d_ntes);
        }
        if (d_tes.n > 1u) {
            qsort(d_tes.v, d_tes.n, sizeof(oracle_event), ev_cmp_abs_t);
        }
        if (d_ntes.n > 1u) {
            qsort(d_ntes.v, d_ntes.n, sizeof(oracle_event), ev_cmp_abs_t);
        }
        if (d_tes.n != 0u) {
            h = d_tes.v[0].t;
        }
        /* ---- state update by the dense-output function (:800), time, outcome ---- */
        {
            double *tau = (double *)malloc(sizeof(double) * batch), *out = (double *)malloc(sizeof(double) * (size_t)n_eq * batch);
            for (uint32_t l = 0; l < batch; ++l) {
                tau[l] = h;
            }
            SYM(oracle_d_output)(P, batch, tc, tau, out);
            for (uint32_t i = 0; i < n_eq; ++i) {
                state[(size_t)i * batch + lane] = out[(size_t)i * batch + lane];
            }
            free(tau);
            free(out);
        }
        int nf = 0;
        for (uint32_t i = 0; i < n_eq; ++i) {
            nf = nf || !isfinite(state[(size_t)i * batch + lane]);
        }
        const dfl nt = dfl_add((dfl){t_hi[lane], t_lo[lane]}, (dfl){h, 0.});
        t_hi[lane] = nt.hi;
        t_lo[lane] = nt.lo;
        last_h[lane] = h;
        if (!(isfinite(nt.hi) && isfinite(nt.lo)) || nf) {
            outcome[lane] = HY_OUTCOME_ERR_NF_STATE;
        } else {
            /* Cooldowns (:848-865). */
            for (uint32_t k = 0; k < n_te; ++k) {
                const size_t ci = (size_t)lane * n_te + k;
                if (cd_on[ci]) {
                    const double tmpv = cd[2u * ci] + h;
                    if (fabs(tmpv) >= cd[2u * ci + 1u]) {
                        cd_on[ci] = 0;
                    } else {
                        cd[2u * ci] = tmpv;
                    }
                }
            }
            /* Non-terminal events before the first terminal one (:871-876). */
            for (uint32_t k = 0; k < d_ntes.n; ++k) {
                if (d_tes.n != 0u && !(fabs(d_ntes.v[k].t) < fabs(h))) {
                    break;
                }
                if (*n_evs < evs_cap) {
                    evs[*n_evs] = d_ntes.v[k];
                } else {
                    overflow = 1;
                }
                ++*n_evs;
            }
            if (d_tes.n != 0u) {
                const oracle_event te = d_tes.v[0];
                const size_t ci = (size_t)lane * n_te + te.idx;
                cd_on[ci] = 1;
                cd[2u * ci] = 0.;
                cd[2u * ci + 1u] = cooldowns[te.idx] >= 0. ? cooldowns[te.idx] : ed_deduce_cooldown(g_eps, te.abs_der);
                if (*n_evs < evs_cap) {
                    evs[*n_evs] = te;
                } else {
                    overflow = 1;
                }
                ++*n_evs;
                outcome[lane] = -(int64_t)te.idx - 1;
            } else {
                outcome[lane] = h == mdt ? HY_OUTCOME_TIME_LIMIT : HY_OUTCOME_SUCCESS;
            }
        }
        free(d_tes.v);
        free(d_ntes.v);
    }
    free(T);
    free(bc);
    free(poly);
    return overflow ? 2 : 0;
}

#endif

/* Raw jet for the closed-form tests: tape[o * n_uvars + u] for lane `lane` (scalar build only). */
#if ORACLE_W == 1
int oracle_jet_w1(const hy_program_desc *P, uint32_t batch, const double *state, const double *pars, const double *t_hi,
                  uint32_t lane, double *tape_out, int mode)
{
    real_t *T = alloc_tape(P);
    if (T == NULL) {
        return 1;
    }
    ctx_t c = {P, batch, lane, 1, pars, T, mode};
    compute_jet(&c, state, t_hi);
    memcpy(tape_out, T, sizeof(double) * (size_t)P->n_uvars * (P->order + 1u));
    free(T);
    return 0;
}

#endif
