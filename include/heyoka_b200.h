/* heyoka_b200 — C ABI of the H100-native batch Taylor integrator.
 *
 * This is the drop-in boundary for heyoka's taylor_adaptive_batch<double> hot path
 * (bluescarni/heyoka @ 9c91f71). The reference funnels every step through three JIT-compiled C
 * function pointers (include/heyoka/detail/ta_jit_data.hpp:35-43):
 *
 *   void step   (double *state, const double *pars, const double *time, double *h_inout, double *tc_or_null);
 *   void step_cm(..., void *tape);
 *   void d_out_f(double *out, const double *tc, const double *h);
 *
 * called from src/taylor_adaptive_batch.cpp:691-698 (step) and :2288,2324 (dense output). The
 * functions below keep those semantics with three differences: (i) the arrays live in device
 * memory (HBM) owned by an hy_batch, (ii) the per-lane host bookkeeping that follows the JIT call
 * in the reference (double-length time update, finiteness scan, outcome; src/taylor_adaptive_batch.cpp:702-727)
 * and the whole propagate_until() loop (:1372-1527) run inside the kernels, (iii) instead of LLVM IR
 * the Taylor decomposition is lowered to a flat opcode program (hy_program) interpreted by
 * hand-written sm_90a kernels. No LLVM, no JIT, no CPU fallback: every compute entry point fails
 * with HY_ERR_CUDA if no CUDA device is usable.
 *
 * All functions return HY_OK (0) or a negative error code; hy_last_error() returns a thread-local
 * message. No exceptions cross this boundary. All arrays are batch-innermost, exactly like the
 * reference's host layout: state[var * batch + lane], pars[par * batch + lane]
 * (src/taylor_adaptive_batch.cpp:679, src/taylor_01.cpp:227-230), tc[(var * (order + 1) + o) * batch + lane]
 * (src/taylor_00.cpp:574-580).
 */
#ifndef HEYOKA_B200_H
#define HEYOKA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HY_OK 0
#define HY_ERR_INVALID_ARG (-1) /* maps to std::invalid_argument in the C++ shim */
#define HY_ERR_NOT_IMPLEMENTED (-2) /* maps to heyoka::not_implemented_error (include/heyoka/exceptions.hpp:19) */
#define HY_ERR_CUDA (-3) /* CUDA runtime failure / no device */
#define HY_ERR_OVERFLOW (-4) /* maps to std::overflow_error */
#define HY_ERR_CALLBACK (-5) /* a host callback passed to the library asked to abort (it keeps its own exception) */

const char *hy_last_error(void);
const char *hy_version(void);

/* taylor_outcome (include/heyoka/taylor.hpp:142-155): int64, success = -2^32 - 1, ... */
#define HY_OUTCOME_SUCCESS (-4294967297LL)
#define HY_OUTCOME_STEP_LIMIT (-4294967298LL)
#define HY_OUTCOME_TIME_LIMIT (-4294967299LL)
#define HY_OUTCOME_ERR_NF_STATE (-4294967300LL)
#define HY_OUTCOME_CB_STOP (-4294967301LL)

/* ------------------------------------------------------------------------------------------------
 * A. Symbolic front end: opaque expression handles.
 *    Replaces: include/heyoka/expression.hpp (construction API), src/expression_ops.cpp,
 *    src/math/{sum,prod,pow,sin,cos,tanh,exp,log,time}.cpp builders.
 * ---------------------------------------------------------------------------------------------- */
typedef struct hy_ex hy_ex;

hy_ex *hy_ex_num(double v);
hy_ex *hy_ex_var(const char *name);
hy_ex *hy_ex_par(uint32_t idx);
hy_ex *hy_ex_time(void);
/* op: '+', '-', '*', '/' (binary, src/expression_ops.cpp:56-92), 'n' = unary minus (b ignored), '^' = pow. */
hy_ex *hy_ex_binary(char op, const hy_ex *a, const hy_ex *b);
/* name: "sin","cos","tanh","exp","log","sqrt","square","sigmoid","relu" (unary); "sum","prod" (n-ary);
 * "leaky_relu", "relup" (binary: argument, slope as a number). */
hy_ex *hy_ex_func(const char *name, const hy_ex *const *args, uint32_t n_args);
hy_ex *hy_ex_copy(const hy_ex *);
void hy_ex_free(hy_ex *);
/* Writes a NUL-terminated rendering into buf (truncated to buf_len); returns the full length. */
size_t hy_ex_str(const hy_ex *, char *buf, size_t buf_len);
/* Symbolic derivative of e with respect to wrt (a variable or a parameter); NULL on error (hy_last_error()). */
hy_ex *hy_ex_diff(const hy_ex *e, const hy_ex *wrt);

/* Variational ODE system of order 1 (heyoka_b200/var_ode_sys.hpp: layout, names, right-hand sides). The arguments:
 * flags != 0 selects them with HY_VAR_ARGS_* bits (args ignored); flags == 0 takes the n_args expressions of args,
 * state variables and / or parameters, in the order given. The augmented system has *n_out_eq = n_eq * (1 + m)
 * equations and *n_out_args = m arguments. out_lhs / out_rhs / out_args == NULL: only the two counts are written;
 * otherwise they receive *n_out_eq, *n_out_eq and *n_out_args new handles (the caller frees each with hy_ex_free).
 * Order > 1 and the time argument: HY_ERR_NOT_IMPLEMENTED. */
#define HY_VAR_ARGS_VARS 1u
#define HY_VAR_ARGS_PARAMS 2u
#define HY_VAR_ARGS_TIME 4u
int hy_var_ode_sys(const hy_ex *const *lhs, const hy_ex *const *rhs, uint32_t n_eq, uint32_t flags,
                   const hy_ex *const *args, uint32_t n_args, uint32_t order, uint32_t *n_out_eq, uint32_t *n_out_args,
                   hy_ex **out_lhs, hy_ex **out_rhs, hy_ex **out_args);

/* Model builders (src/model/nbody.cpp:53-173, src/model/pendulum.cpp:24-29, src/model/ffnn.cpp:70-142).
 * They fill lhs[i]/rhs[i] (caller frees each with hy_ex_free). */
int hy_model_nbody(uint32_t n, const double *masses, uint32_t n_masses, double G, hy_ex **lhs, hy_ex **rhs /* 6n each */);
int hy_model_pendulum(double g, double l, hy_ex **lhs, hy_ex **rhs /* 2 each */);
/* act: per layer 0 = identity, 1 = tanh, 2 = sin, 3 = exp, 4 = sigmoid, 5 = relu. nn_wb == NULL -> weights/biases are par[0..). */
int hy_model_ffnn(const hy_ex *const *inputs, uint32_t n_in, const uint32_t *nn_hidden, uint32_t n_hidden, uint32_t n_out,
                  const int *act, const double *nn_wb, uint32_t n_wb, hy_ex **out /* n_out */);

/* ------------------------------------------------------------------------------------------------
 * B. Program: the lowered Taylor decomposition.
 *    Replaces: taylor_decompose_sys() src/taylor_01.cpp:847-1008 (host, restated), the compact-mode
 *    call tables of src/taylor_02.cpp:830-953 and the LLVM emission of src/taylor_00/01/02.cpp.
 * ---------------------------------------------------------------------------------------------- */

/* Argument reference: bits 31-30 kind, bits 29-0 index. */
#define HY_REF_VAR 0u /* index of a u variable          */
#define HY_REF_NUM 1u /* index into the constant pool   */
#define HY_REF_PAR 2u /* index of a runtime parameter   */
#define HY_REF(kind, idx) (((uint32_t)(kind) << 30) | (uint32_t)(idx))
#define HY_REF_KIND(r) ((r) >> 30)
#define HY_REF_IDX(r) ((r) & 0x3fffffffu)

/* One elementary operation = the definition of one u variable. The recurrence each opcode runs is
 * documented next to its device implementation (heyoka_b200/csrc/recurrences.cuh) with the reference
 * file:line it restates. Suffix letters give the kinds of (a, b): V = u variable index, N = constant
 * pool index, P = parameter index. */
enum hy_opcode {
    HY_OP_SUM = 0,  /* a = offset into args[], b = number of terms (<= 8 after splitting)      */
    HY_OP_SUM_SQ,   /* a = offset into args[], b = number of terms                             */
    HY_OP_SUB_VV,
    HY_OP_SUB_VN,
    HY_OP_SUB_NV,
    HY_OP_SUB_VP,
    HY_OP_SUB_PV,
    HY_OP_NEG,      /* prod(-1, a)                                                             */
    HY_OP_MUL_VV,
    HY_OP_MUL_NV,   /* a = constant, b = variable                                              */
    HY_OP_MUL_PV,   /* a = parameter, b = variable                                             */
    HY_OP_DIV_VV,
    HY_OP_DIV_NV,
    HY_OP_DIV_PV,
    HY_OP_DIV_VN,
    HY_OP_DIV_VP,
    HY_OP_SQUARE,   /* pow(a, 2)                                                               */
    HY_OP_SQRT,     /* pow(a, 1/2)                                                             */
    HY_OP_POW_VN,   /* pow(a, consts[b]); c = (eval_algo << 8) | n, see HY_POW_*               */
    HY_OP_POW_VP,   /* pow(a, par[b])                                                          */
    HY_OP_SIN,      /* a = argument, c = hidden dependency (the u variable holding cos(a))     */
    HY_OP_COS,      /* a = argument, c = hidden dependency (the u variable holding sin(a))     */
    HY_OP_TANH,     /* a = argument, c = hidden dependency (the u variable holding tanh(a)^2)  */
    HY_OP_EXP,
    HY_OP_LOG,
    HY_OP_TIME,
    HY_OP_CFUNC,    /* all arguments are numbers/params: a = function (hy_cfunc), b = offset into
                       args[], c = number of arguments. Order 0: evaluate; higher orders: 0.
                       (include/heyoka/detail/taylor_common.hpp:88-157)                        */
    HY_OP_SIGMOID,  /* a = argument, c = hidden dependency (the u variable holding sigmoid(a)^2),
                       src/math/sigmoid.cpp:137-179                                            */
    HY_OP_RELU,     /* a = argument, b = constant index of the slope of the leaky ReLU (0 = plain),
                       src/math/relu.cpp:157-176                                               */
    HY_OP_RELUP,    /* derivative of the (leaky) ReLU: a = argument, b = constant index of the slope,
                       src/math/relu.cpp:404-424                                               */
    HY_OP_COUNT
};

/* Order-0 evaluation strategy of pow(x, number), src/math/pow.cpp:292-355. */
#define HY_POW_GENERAL 0u
#define HY_POW_POS_SMALL_INT 1u
#define HY_POW_NEG_SMALL_INT 2u
#define HY_POW_POS_SMALL_HALF 3u
#define HY_POW_NEG_SMALL_HALF 4u

enum hy_cfunc { HY_CF_IDENTITY = 0, HY_CF_SUM, HY_CF_PROD, HY_CF_SUB, HY_CF_DIV, HY_CF_POW, HY_CF_SUM_SQ,
                HY_CF_SIN, HY_CF_COS, HY_CF_TANH, HY_CF_EXP, HY_CF_LOG, HY_CF_SIGMOID, HY_CF_RELU, HY_CF_RELUP };

typedef struct hy_op {
    uint32_t opcode;
    uint32_t a, b, c;
} hy_op;

typedef struct hy_program_desc {
    uint32_t n_eq;     /* number of state variables / equations                                 */
    uint32_t n_uvars;  /* state variables + elementary u variables (ops[i] defines u_{n_eq + i}) */
    uint32_t n_pars;   /* number of runtime parameters                                          */
    uint32_t order;    /* Taylor order p                                                        */
    uint32_t n_args;
    uint32_t n_consts;
    int32_t high_accuracy; /* 0: Horner update, 1: compensated summation (src/taylor_00.cpp:355-460) */
    uint32_t n_ev;     /* number of event equations (terminal events first), 0 if none          */
    const hy_op *ops;        /* n_uvars - n_eq entries, in evaluation order                     */
    const uint32_t *args;    /* argument references for n-ary ops                               */
    const double *consts;    /* constant pool                                                   */
    const uint32_t *sv_defs; /* n_eq references: d(x_i)/dt is a u variable, a number or a param */
    const uint32_t *ev_defs; /* n_ev indices: the u variable (possibly a state variable) holding each event
                                equation (sv_funcs_dc of src/taylor_01.cpp:847-1008); NULL if n_ev == 0 */
} hy_program_desc;

typedef struct hy_program hy_program;

/* taylor_order_from_tol(): max(2, ceil(-ln(tol)/2 + 1)), include/heyoka/detail/taylor_common.hpp:165-191. */
int hy_order_from_tol(double tol, uint32_t *order);

/* Decompose + lower an ODE system x_i' = rhs_i. tol <= 0 selects machine epsilon
 * (src/taylor_adaptive_batch.cpp:237-241). Unsupported functions -> HY_ERR_NOT_IMPLEMENTED. */
int hy_program_from_sys(const hy_ex *const *lhs, const hy_ex *const *rhs, uint32_t n_eq, double tol,
                        int high_accuracy, hy_program **out);
/* The same with event equations (terminal events first): the decomposition of src/taylor_00.cpp:605 taylor_decompose_sys(sys,
 * evs); the program then carries ev_defs and the batch built from it detects events (section E). */
int hy_program_from_sys_ev(const hy_ex *const *lhs, const hy_ex *const *rhs, uint32_t n_eq, const hy_ex *const *evs,
                           uint32_t n_ev, double tol, int high_accuracy, hy_program **out);
/* Build from raw arrays (validated: indices in range, ops only read earlier u variables). */
int hy_program_create(const hy_program_desc *desc, hy_program **out);
/* Borrowed view of the program's arrays (valid until hy_program_destroy). */
int hy_program_get_desc(const hy_program *, hy_program_desc *out);
/* Size of the reference-shaped decomposition, n_eq + n_ops + n_eq (test/taylor_decompose.cpp:38-101). */
uint32_t hy_program_dc_size(const hy_program *);
/* Text dump of the decomposition ("u_5 = prod(u_1, u_3) [deps: ...]"), for diagnostics and tests. */
size_t hy_program_dc_str(const hy_program *, char *buf, size_t buf_len);
/* Algorithmic bytes per lane-step, SURVEY.md §8(d): B_min = 8(2 n_eq + n_pars + 7),
 * B_tape = B_min + 16(n_uvars p + n_eq); flops = double-precision operations per lane-step. */
int hy_program_costs(const hy_program *, double *b_min, double *b_tape, double *flops);
void hy_program_destroy(hy_program *);

/* ------------------------------------------------------------------------------------------------
 * C. Batch: device-resident integrator state + the step / propagate kernels.
 *    Replaces: the JIT'd `step` (src/taylor_00.cpp:712-865), step_impl() bookkeeping
 *    (src/taylor_adaptive_batch.cpp:632-727), propagate_until_impl() (:1136-1534), d_out_f
 *    (src/taylor_01.cpp:1015-1185), i_data buffers (src/detail/i_data.cpp).
 * ---------------------------------------------------------------------------------------------- */
typedef struct hy_batch hy_batch;

/* device < 0: current CUDA device. Allocates state, pars, time (hi/lo), last_h, results, tc, scratch. */
int hy_batch_create(const hy_program *, uint32_t batch, int device, hy_batch **out);
/* The same object sharded over several devices of the box: contiguous blocks of lanes, one per device (devices == NULL:
 * every visible device), each driven by its own host thread; lanes are independent, so the results are bit-identical to
 * a single-device batch, including the reference's global exits of propagate_until(). This is what
 * src/ensemble_propagate.cpp:192-311 does with TBB threads. Every hy_batch_* function takes the result except
 * hy_batch_get_ptrs / _set_stream / _propagate_until_dev / _propagate_grid / _propagate_until_cout. */
int hy_batch_create_multi(const hy_program *, uint32_t batch, const int *devices, uint32_t n_devices, hy_batch **out);
uint32_t hy_batch_n_shards(const hy_batch *); /* 0 for a single-device batch */
int hy_device_count(void);                    /* usable CUDA devices (0 if none) */
void hy_batch_destroy(hy_batch *);
/* Diagnostics: compares the lean correctly-rounded division used inside the N-body kernel with the compiler's IEEE
 * division on n pseudo-random pairs; *mismatches must come back 0 (tests/test_gpu_parity.py). */
int hy_selftest_div(uint64_t n, uint64_t seed, uint64_t *mismatches);

/* Page-locks (cudaHostRegister) / releases a host buffer the caller keeps copying from / to: the reference hands out
 * plain std::vector storage (include/heyoka/taylor.hpp:974-977), the drop-in class pins it in place so that the
 * uploads / downloads of every call run at full PCIe speed. A failure is not fatal (returns HY_ERR_CUDA). */
int hy_host_pin(void *ptr, size_t bytes);
int hy_host_unpin(void *ptr);

/* cudaStream_t on which copies and kernels are enqueued (default: the legacy default stream). */
int hy_batch_set_stream(hy_batch *, void *cuda_stream);
int hy_batch_sync(hy_batch *);

/* Host <-> device copies (any pointer may be NULL = leave untouched / don't fetch). */
int hy_batch_upload(hy_batch *, const double *state, const double *pars, const double *t_hi, const double *t_lo);
int hy_batch_download(hy_batch *, double *state, double *t_hi, double *t_lo, double *last_h);
int hy_batch_download_step_res(hy_batch *, int64_t *outcome, double *h);
int hy_batch_download_prop_res(hy_batch *, int64_t *outcome, double *min_h, double *max_h, uint64_t *n_steps);
int hy_batch_download_tc(hy_batch *, double *tc /* n_eq * (order + 1) * batch */);
/* Restores the Taylor coefficients of the last step (copies of an integrator: src/detail/i_data.cpp:335-352 copies
 * m_tc, so that update_d_output() works on the copy before its first write_tc step). */
int hy_batch_upload_tc(hy_batch *, const double *tc /* n_eq * (order + 1) * batch */);

/* Device pointers of the resident arrays, for zero-copy use (torch / NCCL gathers). tc is allocated lazily
 * (first step / propagate with write_tc, hy_batch_download_tc(), hy_batch_d_output()) and NULL before that. */
typedef struct hy_batch_ptrs {
    double *state, *pars, *t_hi, *t_lo, *last_h, *tc, *d_out;
    int64_t *step_outcome;
    int64_t *prop_outcome;
    double *prop_min_h, *prop_max_h;
    uint64_t *prop_n_steps;
} hy_batch_ptrs;
int hy_batch_get_ptrs(hy_batch *, hy_batch_ptrs *out);

/* One step for every lane. max_delta_t: host array of `batch` signed limits (sign = direction), or
 * NULL for +inf (backward != 0: -inf), like step()/step_backward()/step(vec)
 * (src/taylor_adaptive_batch.cpp:1039-1078). If max_delta_t_on_device != 0 the pointer is a device pointer. */
int hy_batch_step(hy_batch *, const double *max_delta_t, int max_delta_t_on_device, int backward, int write_tc);

/* Propagate every lane to its own final time (double-length t_final = hi + lo; lo may be NULL).
 * max_delta_t: host array of positive per-lane limits or NULL (= +inf). max_steps == 0: unlimited.
 * Per-lane semantics follow src/taylor_adaptive_batch.cpp:1372-1527; see DESIGN.md for the two global
 * exits (non-finite state in any lane, iteration limit), which are reproduced by a bounded re-run.
 * Results: hy_batch_download_prop_res(). */
int hy_batch_propagate_until(hy_batch *, const double *t_final_hi, const double *t_final_lo, const double *max_delta_t,
                             uint64_t max_steps, int write_tc);
/* Same, with device-resident inputs (no host traffic): used by the bench's device-timed leg. */
int hy_batch_propagate_until_dev(hy_batch *, const double *d_t_final_hi, const double *d_t_final_lo,
                                 const double *d_max_delta_t, uint64_t max_steps, int write_tc, int *any_nf_or_limit);

/* propagate_until() on HOST buffers in one call - what a caller holding std::vector mirrors does with hy_batch_upload(),
 * hy_batch_propagate_until(), hy_batch_download() and hy_batch_download_prop_res(): state_in [n_eq][batch], t_hi_in,
 * t_lo_in [batch] are uploaded (pars may be NULL: unchanged); state, t_hi, t_lo, last_h, outcome, min_h, max_h, n_steps
 * receive the results (NULL = not wanted; the outputs may alias the inputs). Taylor coefficients are not written
 * (write_tc = 0). On a batch created by hy_batch_create_multi() every shard runs its transfers and its kernel on its
 * own stream from its own host thread; listing the SAME device k times pipelines the batch through that device in k
 * sub-batches (the copies of one overlap the kernels of the others). Page-lock the arrays (hy_host_pin()) for the
 * copies to be asynchronous. Replaces the host-vector path of taylor_adaptive_batch::propagate_until(),
 * src/taylor_adaptive_batch.cpp:1136-1534. */
int hy_batch_propagate_until_host(hy_batch *, const double *state_in, const double *pars, const double *t_hi_in,
                                  const double *t_lo_in, const double *t_final_hi, const double *t_final_lo,
                                  const double *max_delta_t, uint64_t max_steps, double *state, double *t_hi, double *t_lo,
                                  double *last_h, int64_t *outcome, double *min_h, double *max_h, uint64_t *n_steps);

/* propagate_grid() (src/taylor_adaptive_batch.cpp:1545-2055): dense-output sampling on per-lane time grids.
 * grid[k * batch + lane], k < n_pts: finite, strictly monotonic with the same direction in every lane, and
 * grid[lane] == current time (hi part) of the lane. out[(k * n_eq + var) * batch + lane] receives the state at
 * grid point k; entries not reached (early exit: step limit, non-finite state) are NaN. The integrator ends at
 * the last grid point with outcome time_limit; results via hy_batch_download_prop_res(). host arrays. Any number of
 * shards: they run the loop in lock-step and give the bits of the single-device batch. */
int hy_batch_propagate_grid(hy_batch *, const double *grid, uint64_t n_pts, const double *max_delta_t,
                            uint64_t max_steps, double *out);

/* The argument checks of propagate_grid() alone (src/taylor_adaptive_batch.cpp:1575-1670; the current times are those
 * last uploaded): used by the front ends' host loop for integrators with events. */
int hy_batch_check_grid(hy_batch *, const double *grid, uint64_t n_pts, const double *max_delta_t);

/* Continuous output (include/heyoka/continuous_output.hpp, producer src/taylor_adaptive_batch.cpp:1246-1346):
 * hy_batch_propagate_until_cout() runs propagate_until() as the reference's lock-step loop and records, at every
 * iteration, the Taylor coefficients and the (double-length) times of all lanes in device memory. *out is NULL if
 * no iteration completed (non-finite state at the first step). The object is independent of the batch afterwards.
 * hy_cout_eval(): state at per-lane times tm[batch] -> out[n_eq * batch] (host arrays); times outside the
 * integration range use the first / last step's coefficients, like the reference. */
typedef struct hy_cout hy_cout;
int hy_batch_propagate_until_cout(hy_batch *, const double *t_final_hi, const double *t_final_lo,
                                  const double *max_delta_t, uint64_t max_steps, hy_cout **out);
/* Same with a STEP CALLBACK (propagate_until(kw::c_output = true, kw::callback = ...), src/taylor_adaptive_batch.cpp:
 * 1476-1500): after every recorded iteration the stream is synchronised and cb(user) runs on the host - the batch is
 * consistent, the caller may download / upload state and parameters (not the time) from inside it. Return value: > 0
 * continue, 0 stop (every outcome becomes cb_stop, the iteration stays recorded), < 0 abort with HY_ERR_CALLBACK. */
typedef int (*hy_step_callback)(void *user);
int hy_batch_propagate_until_cout_cb(hy_batch *, const double *t_final_hi, const double *t_final_lo,
                                     const double *max_delta_t, uint64_t max_steps, hy_step_callback cb, void *user,
                                     hy_cout **out);
/* A recording driven by the caller's own lock-step loop over hy_batch_step(..., write_tc = 1) (integrators with events:
 * their callbacks are host code; update_c_out(), src/taylor_adaptive_batch.cpp:1320-1346): begin() notes the starting
 * times, append() the Taylor coefficients of the state variables and the times after an iteration, finish() builds the
 * continuous output (forward[lane] != 0: the lane moves forwards in time; *out = NULL if nothing was recorded) and
 * destroys the recorder; destroy() abandons it. */
typedef struct hy_cout_rec hy_cout_rec;
int hy_cout_rec_begin(hy_batch *, hy_cout_rec **out);
int hy_cout_rec_append(hy_batch *, hy_cout_rec *);
int hy_cout_rec_finish(hy_batch *, hy_cout_rec *, const unsigned char *forward, hy_cout **out);
void hy_cout_rec_destroy(hy_cout_rec *);
int hy_cout_eval(hy_cout *, const double *tm, double *out);
/* Per-lane time range [lb, ub] covered (the initial and the final time), number of recorded iterations. */
int hy_cout_get_bounds(const hy_cout *, double *lb, double *ub);
uint64_t hy_cout_n_steps(const hy_cout *);
/* The recorded data on the host, in the reference's layouts (get_times() / get_tcs(), src/continuous_output.cpp:
 * 1157-1169): times_hi / times_lo[(n_steps + 2) * batch] (row 0 = the starting times, row k = the times after
 * iteration k, last row = the +-infinity padding of the binary search), tcs[n_steps][n_eq][order + 1][batch]. NULL
 * pointers are skipped. */
int hy_cout_download(const hy_cout *, double *times_hi, double *times_lo, double *tcs);
void hy_cout_destroy(hy_cout *);

/* Dense output from the last written tc: out[var * batch + lane] = sum_o tc[var][o][lane] * tau[lane]^o
 * (src/taylor_01.cpp:1015-1185; tau relative to the start of the last step). out/tau are host arrays. */
int hy_batch_d_output(hy_batch *, const double *tau, double *out);

/* Taylor map of a variational batch of order 1 (hy_var_ode_sys()): with the current state x (rows 0..n_orig_sv) and
 * state-transition matrix Phi (rows n_orig_sv.., component-major), out[i * batch + lane] = x_i + sum_j Phi_ij dx_j for
 * dx[j * batch + lane], j < n_args. Requires n_orig_sv * (1 + n_args) == n_eq. The sum starts from x_i and adds the
 * rounded products in the order j = 0 .. n_args - 1, each rounded, with no contraction. on_device != 0: dx and out are
 * device pointers (not available on a multi-device batch), the kernel is enqueued on the batch's stream and the call
 * returns without waiting (hy_batch_sync()); else host arrays, and the call returns with out written. */
int hy_batch_eval_taylor_map(hy_batch *, uint32_t n_orig_sv, uint32_t n_args, const double *dx, double *out,
                             int on_device);

/* ------------------------------------------------------------------------------------------------
 * E. Event detection in batch mode.
 *    Replaces: taylor_add_adaptive_step_with_events() (src/taylor_00.cpp:593-710, the JIT'd stepper that returns the jet
 *    of the state variables and of the event equations), the events branch of step_impl()
 *    (src/taylor_adaptive_batch.cpp:728-1035) minus the callbacks, ed_data_batch<T>::detect_events()
 *    (src/detail/event_detection.cpp:1733-2173) with its JIT'd helpers fex_check / poly_rtscc / poly_translate_1
 *    (include/heyoka/detail/ed_data.hpp). A program built by hy_program_from_sys_ev() gives a batch whose every
 *    hy_batch_step() is an event step: jet (Taylor coefficients always written; rows n_eq.. of the device tc array hold
 *    the event equations), detection, propagation cut at the first terminal event of each lane, cooldowns. Callbacks are
 *    the caller's: it reads the detected events back and patches the outcome of a terminal event whose callback asks to
 *    continue (-idx - 1 -> idx). hy_batch_propagate_until{,_host,_dev,_cout,_cout_cb}() and hy_batch_propagate_grid()
 *    refuse such a batch: it is propagated by hy_batch_propagate_until_ev() / hy_batch_propagate_grid_ev() below, or by
 *    a caller's own lock-step loop over hy_batch_step() (the front ends' loop for a step callback together with events).
 * ---------------------------------------------------------------------------------------------- */
typedef struct hy_event_rec {
    uint32_t lane;    /* batch index                                                         */
    uint32_t idx;     /* index among the terminal (terminal != 0) or the non-terminal events  */
    int32_t terminal;
    int32_t d_sgn;    /* sign of the time derivative of the event equation at the event       */
    double t;         /* time of the event relative to the BEGINNING of the step              */
    double abs_der;
} hy_event_rec;
/* The first n_te event equations of the program are terminal. dirs[n_ev] in {-1, 0, 1} (event_direction); cooldowns[n_te]
 * (< 0: automatic, src/detail/event_detection.cpp:519-550); tol: the integrator's tolerance (g_eps of :746-773). */
int hy_batch_set_events(hy_batch *, uint32_t n_te, const int32_t *dirs, const double *cooldowns, double tol);
/* Events of the last step, ready for the callbacks: lanes ascending; per lane the non-terminal events that precede the
 * first terminal one, in time order, then that terminal event. */
uint32_t hy_batch_n_events(const hy_batch *);
int hy_batch_get_events(const hy_batch *, hy_event_rec *out, uint32_t cap);
/* Taylor coefficients of the event equations of the last step, out[n_ev * (order + 1) * batch] (host). */
int hy_batch_download_tc_events(hy_batch *, double *out);
/* reset_cooldowns() / reset_cooldowns(i) (src/taylor_adaptive_batch.cpp:2300-2330): lane < 0 = every lane. */
int hy_batch_reset_cooldowns(hy_batch *, int64_t lane);
/* Cooldown state [n_te][batch]: active flag, time spent in cooldown, cooldown (host arrays). */
int hy_batch_get_cooldowns(hy_batch *, uint8_t *active, double *spent, double *cooldown);
/* Restores a cooldown state (copies of an integrator carry the cooldowns of the original: the reference copies
 * m_te_cooldowns, src/detail/event_detection.cpp:1622-1645). */
int hy_batch_set_cooldowns(hy_batch *, const uint8_t *active, const double *spent, const double *cooldown);

/* Propagation of a batch with event equations on the device: the reference's lock-step loop of propagate_until() /
 * propagate_grid() (src/taylor_adaptive_batch.cpp:1372-1527, :1696-2053) over event steps, with the step limits and
 * the bookkeeping kept on the device. The callback runs on the host once per iteration in which some lane has event
 * records, never otherwise. It receives the n_rec records of the whole batch in the order of hy_batch_get_events()
 * (lanes ascending; per lane the non-terminal events by |t|, then the terminal one), with t_hi / t_lo[k] the absolute
 * time of record k (time after the step - last_h + t, in double-length arithmetic). For every terminal record k it sets
 * cont[k] != 0 to continue (outcome -idx - 1 -> idx) or leaves 0 to stop; the other bytes are ignored. Return value:
 * > 0 go on, < 0 abort with HY_ERR_CALLBACK (the decisions written so far are applied; the iteration's bookkeeping is
 * not done, and an abort in the first iteration leaves the per-lane results at outcome 0, min_h = max_h = 0, 0 steps).
 * The batch is synchronised while the callback runs: it may download / upload state and parameters (not the time).
 * Exits as in the reference: a non-finite state in any lane (after that iteration's bookkeeping), a stopping terminal
 * event in any lane (a terminal record left at 0), max_steps iterations (every outcome becomes step_limit), every lane
 * at its target. The Taylor coefficients are always written. The angle reducer (hy_batch_set_angles()) is refused.
 * hy_batch_propagate_until_ev(): any number of shards; c_out (may be NULL) receives the continuous output of the call
 * (single device only), *c_out = NULL if no iteration completed. Results via hy_batch_download_prop_res().
 * hy_batch_propagate_grid_ev(): any number of shards; the initial propagation to grid[0] runs the same loop with the
 * same callback; out[n_pts * n_eq * batch] as hy_batch_propagate_grid(). */
typedef int (*hy_event_callback)(void *user, const hy_event_rec *recs, const double *t_hi, const double *t_lo,
                                 uint32_t n_rec, unsigned char *cont);
int hy_batch_propagate_until_ev(hy_batch *, const double *t_final_hi, const double *t_final_lo,
                                const double *max_delta_t, uint64_t max_steps, hy_event_callback cb, void *user,
                                hy_cout **c_out);
int hy_batch_propagate_grid_ev(hy_batch *, const double *grid, uint64_t n_pts, const double *max_delta_t,
                               uint64_t max_steps, hy_event_callback cb, void *user, double *out);

/* The angle reducer (callback::angle_reducer, include/heyoka_b200/callback.hpp). hy_batch_set_angles() sets the state
 * variables (indices into the state rows) that the propagate entry points reduce into [0, 2pi) after every step, on
 * the device, where their values are finite: hy_batch_propagate_until{,_host,_dev}(), hy_batch_propagate_grid() (not
 * its initial propagation to the first grid point) and hy_batch_propagate_until_cout{,_cb}(). hy_batch_step() never
 * reduces. n = 0 clears the list; an index out of range or repeated: HY_ERR_INVALID_ARG. The list applies to every
 * shard. With the N-body or dense-network kernel selected (tape_mode 6 to 9), the propagate entry points refuse a
 * non-empty list with HY_ERR_NOT_IMPLEMENTED.
 * hy_reduce_angles() applies the same reduction to n host values in place, with the same bits. */
int hy_batch_set_angles(hy_batch *, const uint32_t *sv_idx, uint32_t n);
int hy_reduce_angles(double *x, uint64_t n);

/* Kernel launch statistics since creation (bench.py's gpu_launches). */
int hy_batch_launch_count(const hy_batch *, uint64_t *n_launches);
/* Name + average duration bookkeeping is done by the caller with CUDA events on the batch's stream. */

/* Tuning knobs (0 = keep default): threads per block and blocks per SM of the persistent kernels. */
int hy_batch_set_launch_config(hy_batch *, uint32_t block_threads, uint32_t blocks_per_sm);

/* Kernel selection. tape_mode: 0 = automatic (shared-memory tape when the system's tape fits in an SM's shared
 * memory, else mode 4), 1 = force the one-thread-per-lane HBM-tape kernel, 2 = force the shared-memory kernel (error if it
 * does not fit), 3 = the same as 2 (kept for compatibility), 4 = the same warp-cooperative kernel with the
 * tape in global memory, 5 = idem with a whole CTA (instead of a warp) working on a chunk of lanes; the automatic
 * mode picks 4 or 5 when shared memory is too small; 6 / 7 = the dedicated N-body kernel (warp / CTA teams; error if
 * the program is not N-body-shaped, see csrc/nb_plan.hpp), which the automatic mode prefers whenever the program
 * qualifies (lanes_per_thread is ignored; lanes_per_warp = lanes per team); 8 = the dense-network kernel; 9 = the N-body kernel with one
 * thread per lane (programs with ONE pair interaction, e.g. the two-body problem; the automatic mode takes it when it
 * applies, HEYOKA_B200_NB_LANE=0 turns that off). lanes_per_warp (1..32, power of two) / lanes_per_thread (1, 2 or 4, dividing lanes_per_warp)
 * only apply to the shared-memory kernel; 0 = automatic. block_threads = 32 x warps per block.
 * The environment variable HEYOKA_B200_TAPE=hbm|smem sets the default. */
int hy_batch_set_kernel(hy_batch *, int tape_mode, uint32_t lanes_per_warp, uint32_t lanes_per_thread,
                        uint32_t block_threads, uint32_t blocks_per_sm);
typedef struct hy_kernel_info {
    int32_t tape_mode;            /* 1 = HBM tape (thread per lane), 2 = shared-memory tape, 4 / 5 = cooperative, global tape (warp / CTA teams), 6 / 7 = N-body kernel (warp / CTA teams), 8 = dense-network kernel, 9 = N-body kernel, one thread per lane (one pair interaction) */
    uint32_t lanes_per_warp, lanes_per_thread, block_threads, blocks_per_sm, grid;
    uint64_t smem_bytes;          /* dynamic shared memory per CTA */
    uint32_t tape_slots_per_lane; /* doubles of tape per lane in the selected strategy */
    uint32_t n_segments;          /* dependency levels of the decomposition (cf. src/taylor_02.cpp:105-207) */
    uint32_t n_fused;             /* superinstructions found by the planner (fused N-body pair interactions) */
    uint32_t n_sms;
    uint32_t tmem_cols_per_warp;  /* always 0: sm_90 has no tensor memory (field kept for ABI compatibility) */
    uint32_t reserved;
} hy_kernel_info;
int hy_batch_get_kernel(const hy_batch *, hy_kernel_info *out);

#ifdef __cplusplus
}
#endif

#endif
