// k_nn: the sm_90a kernel for right-hand sides that are dense feed-forward networks, x' = ffnn(x) (nn_plan.hpp;
// BASELINE.json configs[4]: model::ffnn, 3 x 64 tanh, order 15).
//
// A CTA of 256 threads owns LB = 2 lanes and runs their whole propagate_until() loop (persistent, chunks claimed from
// an atomic counter, like k_coop / k_nb). Per Taylor order n and layer:
//   * the layer's linear part z^[n] = W a^[n] (+ b at order 0) is ONE matrix product [n_out x n_in] . [n_in x lanes] on
//     the FP64 tensor cores: mma.sync.aligned.m8n8k4.f64 (SASS DMMA), 8 output neurons per warp and instruction, the
//     lanes in the N dimension, two accumulator chains per tile;
//   * the weights of every layer are staged ONCE per CTA from global to shared memory by the TMA unit (one
//     cp.async.bulk + mbarrier of the host-prepared, bank-conflict-free padded image: SASS UBLKCP), and stay there;
//   * tanh (src/math/tanh.cpp:183-318) and its hidden dependency tanh^2 (src/math/pow.cpp square recurrence) are run by
//     one thread per (neuron, lane) with the reference's sequential summation order. The histories of z, tanh and
//     tanh^2 are [row][order][neuron][lane] arrays in shared memory (tanh^2 is only ever touched by its own thread).
//     The histories are what bounds the lanes per CTA: 3 x 64 tanh at order 15 takes 2 lanes in the 227 KB of an
//     H100 SM;
//   * the output layer's z^[n] are the derivatives of the state variables: x^[n+1] = z^[n] / (n + 1).
// The Taylor coefficients of the state variables live in shared memory too (step size, state update, optional copy to
// the public tc array): apart from state in / state out nothing touches HBM.
// Only the matrix products differ from the generic kernels (same products, different association, fused): a few ulp on
// every z^[n] (tests/test_gpu_nn_shapes.py states the bound against a series reference of the network).
// Divergence from the reference on non-finite states: the matrix product multiplies the zero weights too, and
// 0 * NaN = NaN, whereas the reference never multiplies by a weight the expression builder dropped. So a NaN (or inf)
// in one state variable of a lane reaches every neuron of that lane, every state variable's coefficients of order >= 1,
// its step size and its time. The generic kernels keep the NaN in the state variables whose jet reads it, and their
// step size stays finite unless state variable 0 is one of them. The lane's outcome (err_nf_state) and every other lane
// are the same (tests/test_gpu_nn_shapes.py::test_one_product_nan_lane_in_last_cta).
#ifndef HEYOKA_B200_CSRC_NN_KERNEL_CUH
#define HEYOKA_B200_CSRC_NN_KERNEL_CUH

#include <cstdint>

#include <cuda_runtime.h>

#include "kernels.cuh"

namespace heyoka_b200::dev
{

constexpr int NN_MAX_LAYERS = 8;
constexpr int NN_LB = 2;        // lanes per CTA
constexpr int NN_THREADS = 256; // 8 warps

struct nn_dev_plan {
    const double *wimg;          // padded weights + biases of every layer, exactly as they sit in shared memory
    const std::uint32_t *out_of_sv; // [n_eq]: output neuron of every state variable
    std::uint32_t wimg_doubles;  // multiple of 2
    std::uint32_t n_layers;
    std::uint32_t n_in[NN_MAX_LAYERS], n_out[NN_MAX_LAYERS], act[NN_MAX_LAYERS];
    std::uint32_t n_in_pad[NN_MAX_LAYERS], n_out_pad[NN_MAX_LAYERS]; // multiples of 4 / 8
    std::uint32_t ldw[NN_MAX_LAYERS], w_off[NN_MAX_LAYERS], b_off[NN_MAX_LAYERS]; // doubles, into wimg
    std::uint32_t hist_off[NN_MAX_LAYERS]; // doubles, into the history area: [3][order][n_out][LB] (hidden layers)
    std::uint32_t hist_doubles, max_out;
};

namespace nnk
{

__device__ __forceinline__ void dmma(double &d0, double &d1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(d0), "+d"(d1)
                 : "d"(a), "d"(b));
}
__device__ __forceinline__ void mbar_init(std::uint64_t *bar, unsigned count)
{
    const unsigned a = static_cast<unsigned>(__cvta_generic_to_shared(bar));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(a), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(std::uint64_t *bar, unsigned bytes)
{
    const unsigned a = static_cast<unsigned>(__cvta_generic_to_shared(bar));
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(a), "r"(bytes) : "memory");
}
// TMA bulk copy global -> shared, completion signalled on the mbarrier (bytes: multiple of 16, 16-byte aligned).
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, std::uint64_t *bar)
{
    const unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(dst));
    const unsigned b = static_cast<unsigned>(__cvta_generic_to_shared(bar));
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(d),
                 "l"(src), "r"(bytes), "r"(b)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(std::uint64_t *bar, unsigned parity)
{
    const unsigned a = static_cast<unsigned>(__cvta_generic_to_shared(bar));
    unsigned done = 0;
    while (done == 0u) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done)
                     : "r"(a), "r"(parity)
                     : "memory");
    }
}

} // namespace nnk

template <bool PROP>
__global__ void __launch_bounds__(NN_THREADS, 1) k_nn(program P, nn_dev_plan NP, batch D, run_args R)
{
    constexpr int LB = NN_LB;
    extern __shared__ __align__(16) double smem_raw[];
    const std::uint32_t p = P.order, n_eq = P.n_eq, tid = threadIdx.x, lane_id = tid & 31u, warp = tid >> 5;
    constexpr std::uint32_t n_warps = NN_THREADS / 32;

    // ---- shared memory: weights | histories | state-variable coefficients | output buffer | scalars ----
    double *wimg = smem_raw;
    double *hist = wimg + NP.wimg_doubles;
    double *xc = hist + NP.hist_doubles;                      // [p + 1][n_eq][LB]
    double *outz = xc + static_cast<std::size_t>(p + 1u) * n_eq * LB; // [max_out][LB]
    double *sc = outz + static_cast<std::size_t>(NP.max_out) * LB;    // h[LB], then flags
    double *s_h = sc;
    int *s_run = reinterpret_cast<int *>(sc + LB);            // running[LB]
    unsigned *s_nf = reinterpret_cast<unsigned *>(s_run + LB); // non-finite mask
    __shared__ __align__(8) std::uint64_t wbar;
    __shared__ unsigned int claimed;
    __shared__ lane_prop parked[LB];
    __shared__ double nn_zero;
    if (tid == 0u) {
        nn_zero = 0.;
    }

    // ---- weights: global -> shared through the TMA unit, once per CTA ----
    if (tid == 0u) {
        nnk::mbar_init(&wbar, 1u);
    }
    __syncthreads();
    if (tid == 0u) {
        // (The copy is split in chunks of at most 32 KB; every chunk completes on the same barrier phase.)
        const unsigned total = NP.wimg_doubles * 8u;
        nnk::mbar_expect_tx(&wbar, total);
        for (unsigned off = 0; off < total; off += 32768u) {
            const unsigned bytes = total - off < 32768u ? total - off : 32768u;
            nnk::bulk_g2s(reinterpret_cast<char *>(wimg) + off, reinterpret_cast<const char *>(NP.wimg) + off, bytes,
                          &wbar);
        }
    }
    nnk::mbar_wait(&wbar, 0u);

    const std::uint32_t n_chunks = (D.n + LB - 1u) / LB;
    const bool owner = tid < LB;

    // The jet of the chunk's lanes: fills xc[0..p].
    const auto jet = [&](std::uint32_t lane0) {
        // Order 0: the state.
        for (std::uint32_t it = tid; it < n_eq * LB; it += NN_THREADS) {
            const std::uint32_t sv = it / LB, l = it % LB;
            const std::uint32_t g = lane0 + l < D.n ? lane0 + l : D.n - 1u;
            xc[sv * LB + l] = D.state[static_cast<std::size_t>(sv) * D.n + g];
        }
        __syncthreads();
        for (std::uint32_t n = 0; n < p; ++n) {
            const double *in = xc + static_cast<std::size_t>(n) * n_eq * LB; // a^[n] of the current layer: [n_in][LB]
            for (std::uint32_t L = 0; L < NP.n_layers; ++L) {
                const std::uint32_t n_in = NP.n_in[L], n_out = NP.n_out[L], kpad = NP.n_in_pad[L], ldw = NP.ldw[L];
                const bool hidden = NP.act[L] != 0u;
                double *zh = hist + NP.hist_off[L];                                  // z: [order][n_out][LB]
                double *th = zh + static_cast<std::size_t>(p) * n_out * LB;          // activation output
                double *sh = th + static_cast<std::size_t>(p) * n_out * LB;          // its square
                // ---- z^[n] = W a^[n] (+ b): one 8 x 8 x k tile per warp and pass ----
                {
                    const std::uint32_t row_in_tile = lane_id >> 2, kk = lane_id & 3u;
                    const bool b_ok = row_in_tile < LB; // B fragment: a[k0 + kk][lane = lane_id / 4]
                    for (std::uint32_t m = warp; m * 8u < NP.n_out_pad[L]; m += n_warps) {
                        const double *wr = wimg + NP.w_off[L] + static_cast<std::size_t>(m * 8u + row_in_tile) * ldw + kk;
                        const double *bp = in + kk * LB + row_in_tile;
                        double c0 = 0., c1 = 0., e0 = 0., e1 = 0.;
                        if (n_in == kpad && (kpad & 7u) == 0u) {
                            // Full tiles (the 64-input layers): no tests on k, the B fragment of a thread whose column
                            // carries no lane is read from a zero (stride 0) instead of selected.
                            const double *ap = wr, *bq = b_ok ? bp : &nn_zero;
                            const std::uint32_t bs = b_ok ? 4u * LB : 0u;
                            for (std::uint32_t k0 = 0; k0 < kpad; k0 += 8u) {
                                nnk::dmma(c0, c1, ap[0], bq[0]);
                                nnk::dmma(e0, e1, ap[4], bq[bs]);
                                ap += 8;
                                bq += 2u * bs;
                            }
                        } else
                        for (std::uint32_t k0 = 0; k0 < kpad; k0 += 8u) {
                            const double a0 = wr[k0];
                            const double b0 = (b_ok && k0 + kk < n_in) ? bp[k0 * LB] : 0.;
                            nnk::dmma(c0, c1, a0, b0);
                            if (k0 + 4u < kpad) {
                                const double a1 = wr[k0 + 4u];
                                const double b1 = (b_ok && k0 + 4u + kk < n_in) ? bp[(k0 + 4u) * LB] : 0.;
                                nnk::dmma(e0, e1, a1, b1);
                            }
                        }
                        c0 += e0;
                        c1 += e1;
                        // C fragment: row = lane_id / 4 (neuron), columns (lane_id % 4) * 2, + 1 (lanes).
                        const std::uint32_t i = m * 8u + row_in_tile, col = kk * 2u;
                        if (i < n_out && col < LB) {
                            const double bias = n == 0u ? wimg[NP.b_off[L] + i] : 0.;
                            double *dst = hidden ? zh + (static_cast<std::size_t>(n) * n_out + i) * LB : outz + i * LB;
                            dst[col] = c0 + bias;
                            if (col + 1u < LB) {
                                dst[col + 1u] = c1 + bias;
                            }
                        }
                    }
                }
                __syncthreads();
                if (hidden) {
                    // ---- tanh and tanh^2, one thread per (neuron, lane) ----
                    const std::uint32_t n_items = n_out * LB;
                    const std::size_t so = static_cast<std::size_t>(n_out) * LB; // stride between orders
                    for (std::uint32_t it = tid; it < n_items; it += NN_THREADS) {
                        const double *zp = zh + it;
                        double *tp = th + it, *sp = sh + it;
                        const double z = zp[n * so];
                        double t = 0.;
                        if (n == 0u) {
                            t = ::tanh(z);
                        } else {
                            // b^[n] - (1/n) sum_{j=1..n} j (c^[n-j] b^[j]), c = tanh(b)^2 (src/math/tanh.cpp:183-318), j
                            // ascending.
                            double acc = 0., jd = 1.;
                            const double *zq = zp + so, *cq = sp + (n - 1u) * so;
                            for (std::uint32_t j = 1; j <= n; ++j) {
                                acc = ::fma(jd, *cq * *zq, acc);
                                jd += 1.;
                                zq += so;
                                cq -= so;
                            }
                            t = z - acc / static_cast<double>(n);
                        }
                        tp[n * so] = t;
                        // Square (src/math/pow.cpp:618-963, exponent 2).
                        double sq = 0.;
                        if (n == 0u) {
                            sq = t * t;
                        } else {
                            const bool odd = (n & 1u) != 0u;
                            const std::uint32_t j1 = odd ? (n - 1u) / 2u : (n - 2u) / 2u;
                            double acc = 0.;
                            const double *pa = tp + n * so, *pb = tp;
                            for (std::uint32_t j = 0; j <= j1; ++j) {
                                acc = ::fma(*pa, *pb, acc);
                                pa -= so;
                                pb += so;
                            }
                            if (odd) {
                                sq = acc + acc;
                            } else {
                                const double h2 = tp[(n / 2u) * so];
                                sq = (acc + acc) + h2 * h2;
                            }
                        }
                        sp[n * so] = sq;
                    }
                    __syncthreads();
                    in = th + static_cast<std::size_t>(n) * n_out * LB;
                } else {
                    // ---- output layer: x^[n+1] = z^[n] / (n + 1) (src/taylor_02.cpp:245-287) ----
                    for (std::uint32_t it = tid; it < n_eq * LB; it += NN_THREADS) {
                        const std::uint32_t sv = it / LB, l = it % LB;
                        xc[(static_cast<std::size_t>(n + 1u) * n_eq + sv) * LB + l]
                            = outz[__ldg(NP.out_of_sv + sv) * LB + l] / static_cast<double>(n + 1u);
                    }
                    __syncthreads();
                }
            }
        }
    };

    // Step size of lane l (reference loop, src/taylor_00.cpp:102-273), owner threads.
    const auto step_size = [&](std::uint32_t l, double max_delta_t) {
        double m0 = fabs(xc[l]), mp = fabs(xc[static_cast<std::size_t>(p) * n_eq * LB + l]),
               mp1 = fabs(xc[static_cast<std::size_t>(p - 1u) * n_eq * LB + l]);
        for (std::uint32_t sv = 1; sv < n_eq; ++sv) {
            m0 = std_max(m0, fabs(xc[sv * LB + l]));
            mp = std_max(mp, fabs(xc[(static_cast<std::size_t>(p) * n_eq + sv) * LB + l]));
            mp1 = std_max(mp1, fabs(xc[(static_cast<std::size_t>(p - 1u) * n_eq + sv) * LB + l]));
        }
        return h_from_norms(P, m0, mp, mp1, max_delta_t);
    };
    // State update + optional copy of the coefficients to the public tc array; lanes with s_run == 0 are left alone.
    const auto update = [&](std::uint32_t lane0) {
        for (std::uint32_t it = tid; it < n_eq * LB; it += NN_THREADS) {
            const std::uint32_t sv = it / LB, l = it % LB, g = lane0 + l;
            if (g < D.n && s_run[l] != 0) {
                const double *c = xc + sv * LB + l;
                const std::size_t so = static_cast<std::size_t>(n_eq) * LB;
                const double res = eval_poly(P, [c, so](std::uint32_t o) { return c[o * so]; }, s_h[l]);
                D.state[static_cast<std::size_t>(sv) * D.n + g] = res;
                if (!isfinite(res)) {
                    atomicOr(s_nf, 1u << l);
                }
                if (R.write_tc != 0) {
                    for (std::uint32_t o = 0; o <= p; ++o) {
                        D.tc[(static_cast<std::size_t>(sv) * (p + 1u) + o) * D.n + g] = c[o * so];
                    }
                }
            }
        }
    };
    const auto claim = [&]() {
        if (tid == 0u) {
            claimed = atomicAdd(R.counter, 1u);
        }
        __syncthreads();
        const unsigned c = claimed;
        __syncthreads();
        return c;
    };

    for (std::uint32_t chunk = claim(); chunk < n_chunks; chunk = claim()) {
        const std::uint32_t lane0 = chunk * LB, lane_raw = lane0 + tid;
        bool valid = owner && lane_raw < D.n;
        const std::uint32_t lane = valid ? lane_raw : D.n - 1u;
        if (tid == 0u) {
            *s_nf = 0u;
        }
        if constexpr (!PROP) {
            if (owner) {
                const bool skipped = R.skip != nullptr && R.skip[lane] != 0u;
                valid = valid && !skipped;
                s_run[tid] = skipped ? 0 : 1;
            }
            __syncthreads();
            jet(lane0);
            double h = 0., mdt = 0.;
            if (owner) {
                mdt = R.max_delta_t != nullptr ? R.max_delta_t[lane] : R.default_max_delta_t;
                h = step_size(tid, mdt);
                s_h[tid] = h;
            }
            __syncthreads();
            update(lane0);
            __syncthreads();
            if (valid) {
                const dfl nt = dfl_add(dfl{D.t_hi[lane], D.t_lo[lane]}, dfl{h, 0.});
                D.t_hi[lane] = nt.hi;
                D.t_lo[lane] = nt.lo;
                D.last_h[lane] = h;
                const bool nf = !(isfinite(nt.hi) && isfinite(nt.lo)) || ((*s_nf >> tid) & 1u) != 0u;
                D.step_outcome[lane]
                    = nf ? HY_OUTCOME_ERR_NF_STATE : (h == mdt ? HY_OUTCOME_TIME_LIMIT : HY_OUTCOME_SUCCESS);
            }
        } else {
            bool running = false;
            if (owner) {
                lane_prop lp;
                lp.init(D, R, lane);
                parked[tid] = lp;
                running = lp.running;
            }
            while (__syncthreads_or(running ? 1 : 0) != 0) {
                if (owner) {
                    s_run[tid] = running ? 1 : 0;
                }
                if (tid == 0u) {
                    *s_nf = 0u;
                }
                __syncthreads();
                jet(lane0);
                double h = 0., cur_max = 0.;
                if (owner) {
                    cur_max = parked[tid].cur_max();
                    h = step_size(tid, cur_max);
                    s_h[tid] = h;
                }
                __syncthreads();
                update(lane0);
                __syncthreads();
                if (running) {
                    lane_prop lp = parked[tid];
                    lp.advance(h, cur_max, ((*s_nf >> tid) & 1u) != 0u, R, valid);
                    parked[tid] = lp;
                    running = lp.running;
                }
            }
            if (valid) {
                parked[tid].store(D, lane);
                parked[tid].report_iters(R);
            }
        }
        __syncthreads();
    }
}

} // namespace heyoka_b200::dev

#endif
