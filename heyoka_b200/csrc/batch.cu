// C ABI, device part (include/heyoka_b200.h section C): device-resident batch state, kernel selection and
// launches. The kernels themselves are in kernels.cuh.
#include <heyoka_b200.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <initializer_list>
#include <limits>
#include <memory>
#include <new>
#include <optional>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include <cuda_runtime.h>

#include "capi_common.hpp"
#include "coop_variants.hpp"
#include "device_program.cuh"
#include "kernels.cuh"
#include "nb_kernel.cuh"
#include "nb_plan.hpp"
#include "nb_variants.hpp"
#include "nn_kernel.cuh"
#include "nn_plan.hpp"
#include "nn_variants.hpp"
#include "small_kernels.cuh"
#include "ev_kernels.cuh"
#include "program.hpp"
#include "smem_plan.hpp"

namespace hy = heyoka_b200;
namespace dev = heyoka_b200::dev;
using hy::detail::cuda_error;
using hy::detail::translate_exception;

#define HY_CUDA_CHECK(expr)                                                                                            \
    do {                                                                                                               \
        const cudaError_t err_ = (expr);                                                                               \
        if (err_ != cudaSuccess) {                                                                                     \
            throw cuda_error(std::string("CUDA error in " #expr ": ") + cudaGetErrorString(err_));                     \
        }                                                                                                              \
    } while (0)

// ------------------------------------------------------------------------------------------------
// Cooperative-kernel dispatch over (lanes per CTA, lanes per thread).
// ------------------------------------------------------------------------------------------------
namespace
{

using hy::detail::coop_variant;

// maxt: upper bound on the threads per CTA the variant was compiled for (256: up to 255 registers per thread).
// mode: 1 = the plan contains elementary ops, 0 = superinstructions only,
// 4 = any plan, tape and tables in global memory, 5 = idem with the whole CTA working on one chunk of lanes.
const coop_variant *find_variant(int L, int N, int maxt, int mode)
{
    const hy::detail::coop_family fams[] = {
        hy::detail::coop_family_n1_512_m1(),
        hy::detail::coop_family_n1_512_m0(),
        hy::detail::coop_family_n1_256_m1(),
        hy::detail::coop_family_n1_256_m0(),
        hy::detail::coop_family_n2_512_m1(),
        hy::detail::coop_family_n2_512_m0(),
        hy::detail::coop_family_n2_256_m1(),
        hy::detail::coop_family_n2_256_m0(),
        hy::detail::coop_family_n4_512_m1(),
        hy::detail::coop_family_n4_512_m0(),
        hy::detail::coop_family_n4_256_m1(),
        hy::detail::coop_family_n4_256_m0(),
        hy::detail::coop_family_n1_512_m4(),
        hy::detail::coop_family_n2_512_m4(),
        hy::detail::coop_family_n1_512_m5(),
        hy::detail::coop_family_n2_512_m5()};
    for (const auto &f : fams) {
        for (std::size_t i = 0; i < f.n; ++i) {
            if (f.v[i].L == L && f.v[i].N == N && f.v[i].maxt == maxt && f.v[i].mode == mode) {
                return f.v + i;
            }
        }
    }
    return nullptr;
}

// The N-body kernel's instantiations (nb_variants.hpp).
const hy::detail::nb_variant *find_nb_variant(int LT, bool cta, bool offchip, int maxt, bool lane = false)
{
    const hy::detail::nb_family fams[] = {hy::detail::nb_family_lt1_cta0(),  hy::detail::nb_family_lt2_cta0(),
                                          hy::detail::nb_family_lt4_cta0(),  hy::detail::nb_family_lt8_cta0(),
                                          hy::detail::nb_family_lt16_cta0(), hy::detail::nb_family_lt32_cta0(),
                                          hy::detail::nb_family_lt1_cta1(),  hy::detail::nb_family_lane()};
    for (const auto &f : fams) {
        for (std::size_t i = 0; i < f.n; ++i) {
            if (f.v[i].LT == LT && f.v[i].cta == cta && f.v[i].offchip == offchip && f.v[i].maxt == maxt
                && f.v[i].lane == lane) {
                return f.v + i;
            }
        }
    }
    return nullptr;
}

// The program tables of the cooperative kernels as one blob of 32-bit words (copied to shared memory by every
// CTA): header (dev::coop_header), ops (8 words per item: opcode, a, b, c, destination row, 3 spare), level
// offsets, n-ary argument table, superinstruction operand tables, constants (doubles), state-variable table
// ({row, right-hand-side reference} per state variable).
std::vector<std::uint32_t> make_plan_blob(const hy::detail::smem_plan &pl, const hy_program &p)
{
    std::vector<std::uint32_t> b(sizeof(dev::coop_header) / 4u, 0u);
    const auto align = [&](std::size_t words) {
        while (b.size() % words != 0u) {
            b.push_back(0u);
        }
    };
    dev::coop_header h{};
    h.n_items = static_cast<std::uint32_t>(pl.ops.size());
    h.n_segments = pl.n_segments;
    h.n_eq = p.n_eq;
    h.n_slots = pl.n_slots;
    h.n_gslots = pl.n_gslots;
    align(4);
    h.off_ops = static_cast<std::uint32_t>(b.size());
    for (std::size_t i = 0; i < pl.ops.size(); ++i) {
        const auto &op = pl.ops[i];
        b.insert(b.end(), {op.opcode, op.a, op.b, op.c, pl.dst[i], pl.svo[i], 0u, 0u});
    }
    h.off_seg = static_cast<std::uint32_t>(b.size());
    b.insert(b.end(), pl.seg_offsets.begin(), pl.seg_offsets.end());
    h.off_args = static_cast<std::uint32_t>(b.size());
    b.insert(b.end(), pl.args.begin(), pl.args.end());
    h.off_aux = static_cast<std::uint32_t>(b.size());
    b.insert(b.end(), pl.aux.begin(), pl.aux.end());
    align(2);
    h.off_consts = static_cast<std::uint32_t>(b.size());
    const auto push_double = [&](double c) {
        std::uint32_t w[2];
        std::memcpy(w, &c, sizeof(double));
        b.push_back(w[0]);
        b.push_back(w[1]);
    };
    for (const double c : p.consts) {
        push_double(c);
    }
    for (const double c : pl.extra_consts) {
        push_double(c);
    }
    align(2);
    // Reciprocals 1 / k (IEEE division on the host) for the exact small-integer divisions.
    h.off_rcp = static_cast<std::uint32_t>(b.size());
    for (std::uint32_t k = 0; k <= p.order + 2u; ++k) {
        const double r = k == 0u ? 0. : 1. / static_cast<double>(k);
        std::uint32_t w[2];
        std::memcpy(w, &r, sizeof(double));
        b.push_back(w[0]);
        b.push_back(w[1]);
    }
    align(4);
    h.off_sv = static_cast<std::uint32_t>(b.size());
    for (std::uint32_t i = 0; i < p.n_eq; ++i) {
        b.insert(b.end(), {pl.sv_rows[i], pl.sv_defs[i], pl.sv_cover[i], pl.sv_parent[i]});
    }
    h.off_svout = static_cast<std::uint32_t>(b.size());
    b.insert(b.end(), pl.svout.begin(), pl.svout.end());
    h.off_svphase = static_cast<std::uint32_t>(b.size());
    h.n_svphase = static_cast<std::uint32_t>(pl.sv_phase.size());
    b.insert(b.end(), pl.sv_phase.begin(), pl.sv_phase.end());
    align(4);
    h.n_words = static_cast<std::uint32_t>(b.size());
    std::memcpy(b.data(), &h, sizeof(h));
    return b;
}

// Shared memory of one warp owning L lanes (must match dev::coop_smem<L>::warp_doubles()).
std::size_t coop_warp_bytes(std::uint32_t n_slots, int L)
{
    const std::size_t l = static_cast<std::size_t>(L);
    return (static_cast<std::size_t>(n_slots) * l + 2u * l + (l + 1u) / 2u + 1u) / 2u * 2u * sizeof(double);
}

// Lets kernels take the largest dynamic shared memory the device allows. The attribute belongs to the function, for
// the whole process: a value that depended on one batch would make the launches of another batch fail.
template <typename F>
void allow_max_smem(std::initializer_list<F> fns, std::size_t smem_optin)
{
    for (const F fn : fns) {
        cudaFuncAttributes a{};
        HY_CUDA_CHECK(cudaFuncGetAttributes(&a, fn));
        HY_CUDA_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           static_cast<int>(smem_optin - a.sharedSizeBytes)));
    }
}

// The kernel a batch runs: what hy_batch_get_kernel() reports (in the order of hy_kernel_info), the entry points, and
// the sizes of the scratch the selection owns.
struct kernel_sel {
    enum family_t { hbm, coop, nb, nn } family = hbm;
    int tape_mode = 0; // as hy_kernel_info::tape_mode reports it
    int L = 0, N = 0;  // lanes per warp (team), lanes per thread
    std::uint32_t threads = 0, per_sm = 0, grid = 0;
    std::size_t smem = 0; // dynamic shared memory per CTA
    std::uint32_t tape_slots = 0;
    // Doubles of global scratch: the tape (k_hbm's slabs, the global or overflow tape of k_coop, k_nb's off-chip rows),
    // and the private per-warp coefficient store (dev::coef_view).
    std::size_t gscratch = 0, cscratch = 0;
    const coop_variant *cv = nullptr;
    const hy::detail::nb_variant *nbv = nullptr;
};

// The cooperative plan and its tables as one blob of 32-bit words.
struct coop_tables {
    hy::detail::smem_plan plan;
    std::vector<std::uint32_t> blob;
    std::size_t bytes = 0; // of the blob, rounded up to 16
};

// A decided selection and the host data its commit uploads (the commit fills in the device pointers of nbd and nnd).
struct candidate {
    kernel_sel k;
    std::optional<coop_tables> tables; // a plan that replaces the batch's (with / without the overflow tape)
    dev::nb_dev_plan nbd{};
    std::vector<hy::detail::nb_role> nb_roles;
    dev::nn_dev_plan nnd{};
    std::vector<double> nn_wimg;
};

} // namespace

// ------------------------------------------------------------------------------------------------
// Host objects: a shard is the device state of one block of lanes on one device; a hy_batch is one or more shards.
// ------------------------------------------------------------------------------------------------
namespace
{

struct shard {
    int device = 0;
    cudaStream_t stream = nullptr;
    std::uint32_t n = 0;
    std::uint32_t n_eq = 0, n_pars = 0, order = 0, n_uvars = 0;
    bool high_accuracy = false;

    // Device copies of the program arrays ("hbm" encoding) ...
    uint4 *d_ops = nullptr;
    std::uint32_t *d_args = nullptr, *d_sv_defs = nullptr;
    double *d_consts = nullptr;
    dev::program prog{};
    // ... and of the cooperative plan.
    hy::detail::smem_plan plan;
    std::uint32_t *d_blob = nullptr;
    std::size_t blob_bytes = 0; // rounded up to 16 bytes
    std::shared_ptr<const hy_program> prog_host; // kept for re-planning
    bool opt_fuse = true, opt_fuse_sv = true;
    int opt_spill = -1; // -1 automatic, 0 never, 1 always
    coop_tables make_tables(bool spill) const;
    void set_tables(coop_tables t);
    void ensure_tc();
    // The dedicated N-body kernel (nb_kernel.cuh): plan, device copies of its tables, device plan of the selected shape.
    hy::detail::nb_plan nbp;
    hy::detail::nb_pair_desc *d_nb_pairs = nullptr;
    hy::detail::nb_role *d_nb_roles = nullptr;
    std::uint32_t opt_nb_threads = 0; // HEYOKA_B200_NB_THREADS: preferred CTA size of the N-body kernel
    double *d_nb_consts = nullptr, *d_nb_fac = nullptr;
    dev::nb_dev_plan nbd{};
    int opt_nb = -1; // -1 automatic, 0 never (HEYOKA_B200_NB=0), 1 preferred
    int opt_nb1 = -1; // one thread per lane for single-pair systems: -1 automatic, 0 never (HEYOKA_B200_NB_LANE=0)
    // The dense-network kernel (nn_kernel.cuh): plan, padded weight image, device plan.
    hy::detail::nn_plan nnp;
    double *d_nn_wimg = nullptr;
    std::uint32_t *d_nn_out = nullptr;
    dev::nn_dev_plan nnd{};
    int opt_nn = -1; // 0: never (HEYOKA_B200_NN=0)

    // Event detection (section E of the C ABI; ev_kernels.cuh). n_ev > 0: the program carries event equations, every
    // step is an event step (jet without propagation + detection + propagation cut at the first terminal event).
    std::uint32_t n_ev = 0;
    dev::ev_args eva{};
    std::vector<void *> ev_allocs;
    void ev_setup(std::uint32_t n_te, const std::int32_t *dirs, const double *cooldowns, double tol);
    std::vector<hy_event_rec> ev_step(const double *max_delta_t, int backward);

    // Resident arrays.
    double *d_state = nullptr, *d_pars = nullptr, *d_t_hi = nullptr, *d_t_lo = nullptr, *d_last_h = nullptr,
           *d_tc = nullptr, *d_d_out = nullptr;
    long long *d_step_outcome = nullptr, *d_prop_outcome = nullptr;
    double *d_prop_min_h = nullptr, *d_prop_max_h = nullptr;
    unsigned long long *d_prop_n_steps = nullptr, *d_prop_iters = nullptr;
    unsigned char *d_skip = nullptr; // per-lane mask of the masked zero-length step (propagate_finish())
    // The angle reducer (hy_batch_set_angles()): per state variable, 1 = reduced into [0, 2pi) after every step of the
    // propagate entry points; angles_on = the list is not empty. The device copy stays allocated once made, so that
    // setting and clearing the list around every propagation costs no allocation.
    std::vector<unsigned char> angles;
    unsigned char *d_angles = nullptr;
    bool angles_on = false;
    const unsigned char *prop_angles() const;

    // Scratch.
    double *d_gscratch = nullptr, *d_cscratch = nullptr; // the selection's (kernel_sel::gscratch, cscratch)
    std::size_t slab_doubles = 0; // one warp's tape slab of k_hbm
    double *d_tmp = nullptr;      // 3 * n doubles: staged per-lane inputs (t_final hi/lo, max_delta_t)
    double *d_snapshot = nullptr; // state + time snapshot for the global-exit replay
    double *d_tmap = nullptr;     // staged dx and out of hy_batch_eval_taylor_map() (host form), allocated on first use
    std::size_t tmap_doubles = 0;
    unsigned int *d_counter = nullptr;
    dev::run_flags *d_flags = nullptr;

    // Kernel selection / launch geometry.
    std::uint32_t n_sms = 0;
    std::size_t smem_per_block_max = 0, smem_per_sm = 0;
    kernel_sel sel;
    std::uint32_t h_threads = 256; // CTA size of k_hbm when a request gives none: the last one given
    std::uint64_t n_launches = 0;

    ~shard();
    void free_all() noexcept;
    dev::batch view() const;
    template <typename T>
    T *dalloc(std::size_t count);
    template <typename T>
    T *dupload(const std::vector<T> &v);
    // Kernel selection: decide() chooses without side effects on the batch, commit() installs the choice.
    candidate decide(int want_mode, int L, int N, std::uint32_t threads, std::uint32_t blocks_per_sm) const;
    void setup_hbm(std::uint32_t threads, std::uint32_t blocks_per_sm, candidate &c) const;
    bool setup_coop(int L, int N, std::uint32_t threads, std::uint32_t ctas_per_sm, candidate &c) const;
    void setup_coop_global(int L, int N, std::uint32_t threads, int cta, candidate &c) const;
    bool setup_nb(int LT, std::uint32_t threads, int want_cta, int want_lane, candidate &c) const;
    bool setup_nn(candidate &c) const;
    std::size_t free_bytes_after_release() const;
    void commit(candidate c);
    void launch(bool prop, const dev::run_args &R);
};

} // namespace

// Lanes [off[i], off[i + 1]) of the batch live on shards[i]; host arrays are batch-innermost ([row][batch]), so a
// shard's slice of a row is contiguous and its copies are pitched 2D copies.
struct hy_batch {
    std::vector<std::unique_ptr<shard>> shards; // at least one
    std::vector<std::uint32_t> off;
    std::uint32_t n = 0, n_eq = 0;
    bool multi = false; // created by hy_batch_create_multi(), whatever its number of shards
    // Events: every shard detects the events of its own lanes; ev_host holds those of the last step for the whole
    // batch, in the order the callbacks must run.
    std::uint32_t n_ev = 0, n_te = 0;
    bool ev_set = false;
    std::vector<hy_event_rec> ev_host;
};

template <typename T>
T *shard::dalloc(std::size_t count)
{
    void *p = nullptr;
    HY_CUDA_CHECK(cudaMalloc(&p, std::max<std::size_t>(count, 1u) * sizeof(T)));
    return static_cast<T *>(p);
}

template <typename T>
T *shard::dupload(const std::vector<T> &v)
{
    T *p = dalloc<T>(v.size());
    if (!v.empty()) {
        HY_CUDA_CHECK(cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    }
    return p;
}

void shard::free_all() noexcept
{
    for (void *p :
         {static_cast<void *>(d_ops), static_cast<void *>(d_args), static_cast<void *>(d_sv_defs),
          static_cast<void *>(d_consts), static_cast<void *>(d_blob), static_cast<void *>(d_gscratch),
          static_cast<void *>(d_cscratch),
          static_cast<void *>(d_state),
          static_cast<void *>(d_pars),
          static_cast<void *>(d_t_hi), static_cast<void *>(d_t_lo), static_cast<void *>(d_last_h),
          static_cast<void *>(d_tc), static_cast<void *>(d_d_out), static_cast<void *>(d_step_outcome),
          static_cast<void *>(d_prop_outcome), static_cast<void *>(d_prop_min_h), static_cast<void *>(d_prop_max_h),
          static_cast<void *>(d_prop_n_steps), static_cast<void *>(d_prop_iters), static_cast<void *>(d_skip),
          static_cast<void *>(d_tmp),
          static_cast<void *>(d_snapshot), static_cast<void *>(d_counter), static_cast<void *>(d_flags),
          static_cast<void *>(d_nb_pairs), static_cast<void *>(d_nb_roles), static_cast<void *>(d_nb_consts),
          static_cast<void *>(d_nb_fac), static_cast<void *>(d_nn_wimg), static_cast<void *>(d_nn_out),
          static_cast<void *>(d_tmap), static_cast<void *>(d_angles)}) {
        if (p != nullptr) {
            cudaFree(p);
        }
    }
    for (void *p : ev_allocs) {
        cudaFree(p);
    }
    ev_allocs.clear();
}

shard::~shard()
{
    int cur = 0;
    if (cudaGetDevice(&cur) == cudaSuccess) {
        cudaSetDevice(device);
        free_all();
        cudaSetDevice(cur);
    }
}

dev::batch shard::view() const
{
    dev::batch b{};
    b.n = n;
    b.state = d_state;
    b.t_hi = d_t_hi;
    b.t_lo = d_t_lo;
    b.last_h = d_last_h;
    b.tc = d_tc;
    b.pars = d_pars;
    b.step_outcome = d_step_outcome;
    b.prop_outcome = d_prop_outcome;
    b.prop_min_h = d_prop_min_h;
    b.prop_max_h = d_prop_max_h;
    b.prop_n_steps = d_prop_n_steps;
    b.prop_iters = d_prop_iters;
    return b;
}

// Device memory that is free once the current selection's scratch is released.
std::size_t shard::free_bytes_after_release() const
{
    std::size_t free_b = 0, total_b = 0;
    HY_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
    return free_b + (sel.gscratch + sel.cscratch) * sizeof(double);
}

void shard::setup_hbm(std::uint32_t threads, std::uint32_t blocks_per_sm, candidate &c) const
{
    if (threads == 0u) {
        threads = h_threads;
    } else if (threads % 32u != 0u || threads > 256u) {
        throw std::invalid_argument("block_threads must be a multiple of 32 not larger than 256");
    }
    if (blocks_per_sm == 0u) {
        int occ = 0;
        HY_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, dev::k_hbm<true>,
                                                                    static_cast<int>(threads), 0));
        blocks_per_sm = static_cast<std::uint32_t>(std::max(occ, 1));
    }

    // One slab per resident warp; never more warps than chunks of 32 lanes.
    const std::uint32_t warps_per_block = threads / 32u;
    const std::uint32_t n_chunks = (n + 31u) / 32u;
    const std::uint32_t needed_blocks = (n_chunks + warps_per_block - 1u) / warps_per_block;
    // The slabs of the resident warps must fit in (half of the free) device memory: large systems (model::ffnn
    // 3 x 64: 43 MB per warp) run with fewer resident blocks rather than failing to allocate.
    const std::size_t per_block = static_cast<std::size_t>(warps_per_block) * slab_doubles * sizeof(double);
    const std::size_t max_blocks
        = std::max<std::size_t>(free_bytes_after_release() / 2u / std::max<std::size_t>(per_block, 1u), 1u);
    const auto grid = static_cast<std::uint32_t>(
        std::min<std::size_t>(std::max(1u, std::min(n_sms * blocks_per_sm, needed_blocks)), max_blocks));
    c.k = {kernel_sel::hbm, 1, 32, 1, threads, blocks_per_sm, grid, 0u, n_uvars * (order + 1u),
           static_cast<std::size_t>(grid) * warps_per_block * slab_doubles};
}

coop_tables shard::make_tables(bool spill) const
{
    coop_tables t;
    t.plan = hy::detail::make_smem_plan(*prog_host, opt_fuse, opt_fuse_sv, spill);
    t.blob = make_plan_blob(t.plan, *prog_host);
    t.bytes = (t.blob.size() + 3u) / 4u * 16u;
    return t;
}

void shard::set_tables(coop_tables t)
{
    if (d_blob != nullptr) {
        HY_CUDA_CHECK(cudaFree(d_blob));
        d_blob = nullptr;
    }
    d_blob = dupload(t.blob);
    blob_bytes = t.bytes;
    plan = std::move(t.plan);
}

// Returns false if the requested / any configuration does not fit in shared memory.
// L = lanes per warp, N = lanes per thread, threads = 32 x warps per block.
bool shard::setup_coop(int L, int N, std::uint32_t threads, std::uint32_t ctas_per_sm, candidate &c) const
{
    const std::size_t reserve = 1024u; // per-block reservation of the driver
    if (N == 0) {
        // Two lanes per thread: the interpreter's per-item overhead is shared and the recurrences get ILP 2.
        N = (L == 0 || L >= 2) ? 2 : 1;
    }
    // Optional overflow tape (HEYOKA_B200_SPILL=1): the superinstructions' private history rows move from shared
    // memory to global memory / L2, which lets 12 instead of 8 warps of the 6-body system reside on an SM.
    // Measured slower (1.89e7 vs 2.47e7 lane-steps/s: the L2 latency lands on the serial pow recurrence), hence
    // off by default; kept because it is what a system slightly too large for shared memory needs.
    if ((opt_spill > 0) != (plan.n_gslots != 0u)) {
        c.tables = make_tables(opt_spill > 0);
    }
    const auto &pl = c.tables ? c.tables->plan : plan;
    const std::size_t blob_sz = c.tables ? c.tables->bytes : blob_bytes;
    if (L == 0) {
        // Lanes per warp: enough of them that an average dependency segment gives work to most of the
        // 32 threads (one work item = one u variable x N lanes), as long as at least 4 warps fit on an SM.
        const double avg_width = static_cast<double>(pl.ops.size()) / std::max(1u, pl.n_segments);
        for (const int cand : {1, 2, 4, 8, 16, 32}) {
            if (cand < N) {
                continue;
            }
            const auto bytes = coop_warp_bytes(pl.n_slots, cand);
            if (blob_sz + bytes + reserve > smem_per_block_max || (smem_per_sm - blob_sz) / bytes < 4u) {
                break;
            }
            L = cand;
            if (avg_width * cand / N >= 12.) {
                break;
            }
        }
        if (L == 0) {
            // Not even 4 warps of the smallest shape fit: take whatever fits at all.
            if (blob_sz + coop_warp_bytes(pl.n_slots, N) + reserve > smem_per_block_max) {
                return false;
            }
            L = N;
        }
    }
    // Warps per CTA that fit next to one copy of the tables (at most 16).
    const auto fit_warps = [&](std::uint32_t n_slots, int lanes) -> std::size_t {
        const auto wb = coop_warp_bytes(n_slots, lanes);
        if (blob_sz + wb + reserve > smem_per_block_max) {
            return 0u;
        }
        return std::min<std::size_t>((smem_per_block_max - reserve - blob_sz) / wb, 16u);
    };
    const auto warp_bytes = coop_warp_bytes(pl.n_slots, L);
    if (blob_sz > 24u * 1024u || blob_sz + warp_bytes + reserve > smem_per_block_max) {
        return false;
    }
    if (threads == 0u) {
        // One CTA per SM holding as many warps as fit in shared memory.
        const std::size_t W = fit_warps(pl.n_slots, L);
        threads = static_cast<std::uint32_t>(32u * std::max<std::size_t>(W, 1u));
    }
    if (threads % 32u != 0u || threads == 0u || threads > 512u) {
        throw std::invalid_argument("Invalid number of threads for the cooperative kernel");
    }
    // Registers: 65536 / 512 threads = 128 per thread, 170 with at most 384 threads, 255 with at most 256.
    int kmode = 0;
    for (const auto &op : pl.ops) {
        kmode = op.opcode < hy::detail::HY_FOP_FIRST ? 1 : kmode;
    }
    // (Not every shape is compiled for every CTA size: fall back to the next larger bound.)
    const int pref_maxt = threads <= 256u ? 256 : 512;
    const coop_variant *v = nullptr;
    for (const int m : {256, 512}) {
        if (m >= pref_maxt && v == nullptr) {
            v = find_variant(L, N, m, kmode);
        }
    }
    if (v == nullptr) {
        throw std::invalid_argument("Unsupported cooperative kernel configuration: " + std::to_string(L)
                                    + " lanes per warp, " + std::to_string(N) + " lanes per thread");
    }
    const std::size_t bytes = blob_sz + static_cast<std::size_t>(threads / 32u) * warp_bytes;
    if (bytes + reserve > smem_per_block_max) {
        return false;
    }
    allow_max_smem({v->step, v->prop}, smem_per_block_max);
    if (ctas_per_sm == 0u) {
        int occ = 0;
        HY_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, v->prop, static_cast<int>(threads), bytes));
        ctas_per_sm = static_cast<std::uint32_t>(std::max(occ, 1));
    }
    const std::uint32_t lanes_per_block = static_cast<std::uint32_t>(L) * (threads / 32u);
    const std::uint32_t n_blocks_needed = (n + lanes_per_block - 1u) / lanes_per_block;
    const std::uint32_t grid = std::max(1u, std::min(n_sms * ctas_per_sm, n_blocks_needed));
    const std::size_t warp_lanes = static_cast<std::size_t>(grid) * (threads / 32u) * static_cast<std::size_t>(L);
    c.k = {kernel_sel::coop, 2, L, N, threads, ctas_per_sm, grid, bytes, pl.n_slots, warp_lanes * pl.n_gslots,
           warp_lanes * (order + 1u) * n_eq, v};
    return true;
}

// The cooperative kernel for systems whose compact tape does not fit in shared memory (model::nbody with 32
// bodies: 56k doubles per lane): same program, same planner, but every warp's tape is a slab of global memory and
// the tables are read in place. Unlike the one-thread-per-lane HBM-tape kernel it fills the GPU with a few
// thousand lanes (a warp works on L lanes, its threads on different u variables).
void shard::setup_coop_global(int L, int N, std::uint32_t threads, int cta, candidate &c) const
{
    c.tables.reset();
    if (plan.n_gslots != 0u) {
        c.tables = make_tables(false);
    }
    const auto &pl = c.tables ? c.tables->plan : plan;
    if (N == 0) {
        N = (L == 0 || L >= 2) ? 2 : 1;
    }
    if (threads == 0u) {
        threads = 512u;
    }
    if (threads % 32u != 0u || threads > 512u) {
        throw std::invalid_argument("Invalid number of threads for the cooperative kernel");
    }
    const std::uint32_t warps = threads / 32u;
    if (cta < 0) {
        // Whole CTAs per chunk of lanes (mode 5) when the levels are wide enough to give work to hundreds of
        // threads and there are too few lanes to keep every warp of the GPU busy for long: the lane-step latency
        // drops by the number of warps (a slow lane no longer holds the launch), and the tapes in flight
        // (n_sms x L lanes) nearly fit in L2. Otherwise one warp per chunk (mode 4).
        const double avg_width = static_cast<double>(pl.ops.size()) / std::max(1u, pl.n_segments);
        const std::uint64_t warp_chunks = (n + static_cast<std::uint32_t>(N) - 1u) / static_cast<std::uint32_t>(N);
        cta = (avg_width >= 128. && warp_chunks < 8ull * n_sms * warps) ? 1 : 0;
    }
    if (L == 0) {
        L = N;
        if (cta == 0) {
            // As many lanes per warp as still leave a chunk of lanes for every resident warp.
            while (2 * L <= 8 && n / static_cast<std::uint32_t>(2 * L) >= n_sms * 16u) {
                L *= 2;
            }
        }
    }
    const auto *v = find_variant(L, N, 512, cta != 0 ? 5 : 4);
    if (v == nullptr) {
        throw std::invalid_argument("Unsupported cooperative kernel configuration (global tape): "
                                    + std::to_string(L) + " lanes per warp, " + std::to_string(N)
                                    + " lanes per thread");
    }
    // Teams (warps, or whole CTAs) per block, each with its own slab and private coefficient store.
    const std::uint32_t teams = cta != 0 ? 1u : warps;
    const std::size_t team_bytes = coop_warp_bytes(pl.n_slots, L);
    const std::uint32_t lanes_per_block = static_cast<std::uint32_t>(L) * teams;
    const std::uint32_t n_blocks_needed = (n + lanes_per_block - 1u) / lanes_per_block;
    const std::size_t max_blocks = std::max<std::size_t>(free_bytes_after_release() / 2u / (team_bytes * teams), 1u);
    const auto grid = static_cast<std::uint32_t>(
        std::max<std::size_t>(1u, std::min<std::size_t>({n_sms, n_blocks_needed, max_blocks})));
    const std::size_t team_count = static_cast<std::size_t>(grid) * teams;
    c.k = {kernel_sel::coop, cta != 0 ? 5 : 4, L, N, threads, 1u, grid, 0u, pl.n_slots,
           team_count * (team_bytes / sizeof(double)), team_count * (order + 1u) * n_eq * L, v};
}

// The table of the one-thread-per-lane N-body kernel (nb1_kernel.cuh) for a plan with ONE pair interaction whose six
// positions each belong to a velocity driven by a single pair output of the same coordinate, or by a number. Returns
// false for anything else (such plans run on k_nb with 32 lanes per warp).
static bool make_nb1_tab(const hy::detail::nb_plan &pl, std::uint32_t n_eq, std::uint32_t order, dev::nb1_tab &tab)
{
    if (!pl.ok || pl.pairs.size() != 1u || pl.sums.size() != 6u || pl.level_offsets.size() != 2u || n_eq != 12u
        || order < 4u) {
        return false;
    }
    const auto &pr = pl.pairs[0];
    bool seen[12] = {};
    std::uint32_t kinds[6];
    for (std::uint32_t s = 0; s < 6u; ++s) {
        const std::uint32_t k = s % 3u, ps = s < 3u ? pr.pa[k] : pr.pb[k];
        const hy::detail::nb_sum_desc *sd = nullptr;
        for (const auto &cand : pl.sums) {
            if (cand.kind != 0u && cand.pos == ps + 1u) {
                if (sd != nullptr) {
                    return false;
                }
                sd = &cand;
            }
        }
        if (sd == nullptr || (sd->out >> 16) == 0u || ps >= pl.pos_sv.size()) {
            return false;
        }
        tab.v_sv[s] = sd->out & 0xffffu;
        tab.x_sv[s] = (sd->out >> 16) - 1u;
        if (tab.x_sv[s] != pl.pos_sv[ps] || tab.v_sv[s] >= 12u || tab.x_sv[s] >= 12u || seen[tab.v_sv[s]]
            || seen[tab.x_sv[s]]) {
            return false;
        }
        seen[tab.v_sv[s]] = seen[tab.x_sv[s]] = true;
        if (tab.v_sv[s] == 0u || tab.x_sv[s] == 0u) {
            tab.sv0_slot = s;
            tab.sv0_is_x = tab.x_sv[s] == 0u ? 1u : 0u;
        }
        if (sd->kind == 2u) {
            // (Only the right-hand side +0: what model::nbody produces for a body that nothing pulls on.)
            if (sd->cidx >= pl.consts.size() || pl.consts[sd->cidx] != 0. || std::signbit(pl.consts[sd->cidx])) {
                return false;
            }
            kinds[s] = 2u;
        } else if (sd->kind == 1u && sd->n_terms == 1u && sd->terms[0] == pr.om[k]) {
            kinds[s] = 0u;
        } else if (sd->kind == 1u && sd->n_terms == 1u && pr.on[k] != 0xffffu && sd->terms[0] == pr.on[k]) {
            kinds[s] = 1u;
        } else {
            return false;
        }
    }
    for (std::uint32_t side = 0; side < 2u; ++side) {
        if (kinds[3u * side] != kinds[3u * side + 1u] || kinds[3u * side] != kinds[3u * side + 2u]) {
            return false;
        }
        tab.kind[side] = kinds[3u * side];
    }
    return true;
}

// The dedicated N-body kernel. LT = lanes per team (0: as many as give every thread of a warp one pair interaction),
// threads = CTA size (0: as many warps as fit; HEYOKA_B200_NB_THREADS caps it), want_cta: -1 automatic.
// Returns false if the program does not qualify or nothing fits.
bool shard::setup_nb(int LT, std::uint32_t threads, int want_cta, int want_lane, candidate &c) const
{
    if (!nbp.ok) {
        return false;
    }
    const std::size_t reserve = 1024u;
    const std::uint32_t n_pairs = static_cast<std::uint32_t>(nbp.pairs.size());
    const std::uint32_t npp = (order + 1u) / 2u;
    const bool cta = want_cta > 0 || (want_cta < 0 && n_pairs > 32u);
    if (!cta && n_pairs > 32u) {
        return false;
    }
    if (LT == 0) {
        LT = 1;
        if (!cta) {
            while (static_cast<std::uint32_t>(2 * LT) * n_pairs <= 32u) {
                LT *= 2;
            }
        }
    }
    if (cta && (LT != 1 || n_pairs > 512u)) {
        return false;
    }
    if (!cta && (LT < 1 || LT > 32 || (LT & (LT - 1)) != 0 || static_cast<std::uint32_t>(LT) * n_pairs > 32u)) {
        return false;
    }
    // One pair interaction, 32 lanes per warp: one thread per lane, nothing exchanged (nb1_kernel.cuh).
    dev::nb1_tab l1{};
    const bool lane = want_lane != 0 && !cta && LT == 32 && make_nb1_tab(nbp, n_eq, order, l1);
    if (want_lane > 0 && !lane) {
        return false;
    }
    const std::uint32_t TT = cta ? 512u : 32u, NL = LT >= 2 ? 2u : 1u;
    // The role records address the outputs in 16-bit units of 16 bytes.
    if (static_cast<std::uint64_t>(nbp.n_out) * LT >= 0xffffu || static_cast<std::uint64_t>(nbp.n_pos) * LT >= 0xffffu) {
        return false;
    }
    auto roles = hy::detail::make_nb_roles(nbp, TT, static_cast<std::uint32_t>(LT), NL);
    if (roles.n_rounds > 32u) {
        return false;
    }
    if (lane) {
        roles = hy::detail::nb_roles{};
    }
    const auto shared_doubles = [&](bool roles_in_smem) {
        std::size_t d = static_cast<std::size_t>(order + 1u) * nbp.fac_stride + ((order + 5u) & ~1u)
                        + ((nbp.consts.size() + 1u) & ~std::size_t(1));
        if (roles_in_smem) {
            d += roles.table.size() * 4u;
        }
        return d;
    };
    const auto team_slots = [&](bool offchip) {
        // (The one-thread-per-lane kernel keeps positions, pair outputs and norms in registers.)
        const std::size_t d = (lane ? 0u : (static_cast<std::size_t>(nbp.n_pos) + nbp.n_out) * LT * 2u)
                              + static_cast<std::size_t>(offchip ? 2u : 5u) * npp * TT * 2u
                              + (3u * hy::detail::nb_norm_copies(static_cast<std::uint32_t>(LT)) + 16u) * LT; // (+ norms, parked bookkeeping)
        return static_cast<std::uint32_t>((d + LT - 1u) / LT);
    };
    // Teams (warps) per CTA that fit in shared memory. CTA teams whose five private rows per thread do not fit keep
    // three of them (r^2, d_2, r^alpha) off chip, in a per-CTA slab of global memory that stays in L2.
    struct choice {
        bool offchip = false, roles_in_smem = false;
        std::uint32_t warps = 0;
    };
    const auto fit = [&](bool offchip) {
        choice c;
        c.offchip = offchip;
        for (const bool ris : {true, false}) {
            const std::size_t sh = shared_doubles(ris) * sizeof(double);
            const std::size_t tb = coop_warp_bytes(team_slots(offchip), LT);
            if (sh + tb + reserve > smem_per_block_max) {
                continue;
            }
            std::uint32_t w = cta ? 16u
                                  : static_cast<std::uint32_t>(
                                        std::min<std::size_t>((smem_per_block_max - reserve - sh) / tb, 16u));
            if (cta && w < 16u) {
                w = 0u;
            }
            if (w > c.warps) {
                c.warps = w;
                c.roles_in_smem = ris;
            }
            if (w != 0u) {
                break;
            }
        }
        return c;
    };
    choice pick = fit(false);
    if (cta && pick.warps == 0u) {
        pick = fit(true);
    }
    if (pick.warps == 0u) {
        return false;
    }
    if (threads == 0u) {
        // Warp teams: 12 warps by default (168 registers per thread: the pair interaction's working set fits without
        // spilling; measured faster than 16 warps of 128 registers and than 8 of 255).
        threads = 32u * (cta ? pick.warps : std::min(pick.warps, 12u));
        if (!cta && opt_nb_threads != 0u) {
            threads = opt_nb_threads;
        }
    }
    if (!cta) {
        threads = std::min(threads, 32u * pick.warps); // (a tuning knob: clamped to what fits)
    }
    if (threads % 32u != 0u || threads == 0u || threads / 32u > pick.warps || (cta && threads != 512u)) {
        throw std::invalid_argument("Invalid number of threads for the N-body kernel");
    }
    const int pref_maxt = threads <= 256u ? 256 : (threads <= 384u ? 384 : 512);
    const hy::detail::nb_variant *v = nullptr;
    for (const int mt : {256, 384, 512}) {
        if (mt >= pref_maxt && v == nullptr) {
            v = find_nb_variant(LT, cta, pick.offchip, mt, lane);
        }
    }
    if (v == nullptr) {
        return false;
    }
    dev::nb_dev_plan &d = c.nbd;
    d.n_pairs = n_pairs;
    d.n_pos = nbp.n_pos;
    d.n_out = nbp.n_out;
    d.n_consts = static_cast<std::uint32_t>(nbp.consts.size());
    d.npp = npp;
    d.fac_stride = nbp.fac_stride;
    d.n_rounds = roles.n_rounds;
    d.round_level_end = roles.round_level_end;
    d.alpha = nbp.alpha;
    d.pow_algo = nbp.pow_algo;
    d.roles_in_smem = pick.roles_in_smem ? 1u : 0u;
    d.shared_doubles = static_cast<std::uint32_t>(shared_doubles(pick.roles_in_smem));
    d.n_slots_equiv = team_slots(pick.offchip);
    d.l1 = l1;
    const std::size_t team_bytes = coop_warp_bytes(d.n_slots_equiv, LT);
    d.team_doubles = static_cast<std::uint32_t>(team_bytes / sizeof(double));
    c.nb_roles = std::move(roles.table);
    const std::uint32_t teams = cta ? 1u : threads / 32u;
    const std::size_t bytes = static_cast<std::size_t>(d.shared_doubles) * sizeof(double) + teams * team_bytes;
    allow_max_smem({v->step, v->prop}, smem_per_block_max);
    const std::uint32_t lanes_per_block = static_cast<std::uint32_t>(LT) * teams;
    const std::uint32_t n_blocks_needed = (n + lanes_per_block - 1u) / lanes_per_block;
    const std::uint32_t grid = std::max(1u, std::min(n_sms, n_blocks_needed));
    c.k = {kernel_sel::nb, lane ? 9 : (cta ? 7 : 6), LT, LT >= 2 ? 2 : 1, threads, 1u, grid, bytes, d.n_slots_equiv,
           pick.offchip ? static_cast<std::size_t>(grid) * npp * 3u * TT * 2u : 0u,
           static_cast<std::size_t>(grid) * teams * (order + 1u) * n_eq * static_cast<std::size_t>(LT), nullptr, v};
    return true;
}

// The dense-network kernel: the padded shared-memory image of the weights is prepared here (row pitch = 4 mod 16
// doubles: the 8 x 4 A fragments of the tensor-core products then read conflict-free), copied once per CTA by the TMA
// unit. Returns false if the program is not a network or does not fit in shared memory.
bool shard::setup_nn(candidate &c) const
{
    if (!nnp.ok || nnp.layers.size() > static_cast<std::size_t>(dev::NN_MAX_LAYERS)) {
        return false;
    }
    dev::nn_dev_plan d{};
    std::vector<double> img;
    std::uint32_t hist = 0, max_out = 0;
    d.n_layers = static_cast<std::uint32_t>(nnp.layers.size());
    for (std::uint32_t l = 0; l < d.n_layers; ++l) {
        const auto &L = nnp.layers[l];
        d.n_in[l] = L.n_in;
        d.n_out[l] = L.n_out;
        d.act[l] = static_cast<std::uint32_t>(L.act);
        d.n_in_pad[l] = (L.n_in + 3u) & ~3u;
        d.n_out_pad[l] = (L.n_out + 7u) & ~7u;
        std::uint32_t ldw = d.n_in_pad[l];
        while (ldw % 16u != 4u) {
            ++ldw;
        }
        d.ldw[l] = ldw;
        d.w_off[l] = static_cast<std::uint32_t>(img.size());
        img.resize(img.size() + static_cast<std::size_t>(d.n_out_pad[l]) * ldw, 0.);
        for (std::uint32_t r = 0; r < L.n_out; ++r) {
            for (std::uint32_t c = 0; c < L.n_in; ++c) {
                img[d.w_off[l] + static_cast<std::size_t>(r) * ldw + c] = L.w[static_cast<std::size_t>(r) * L.n_in + c];
            }
        }
        d.b_off[l] = static_cast<std::uint32_t>(img.size());
        img.insert(img.end(), L.bias.begin(), L.bias.end());
        img.resize((img.size() + 1u) & ~std::size_t(1), 0.);
        d.hist_off[l] = hist;
        if (L.act != 0) {
            hist += 3u * order * L.n_out * dev::NN_LB; // z, the activation and its square
        }
        max_out = std::max(max_out, L.n_out);
    }
    d.wimg_doubles = static_cast<std::uint32_t>(img.size());
    d.hist_doubles = hist;
    d.max_out = max_out;
    const std::size_t doubles = img.size() + hist + static_cast<std::size_t>(order + 1u) * n_eq * dev::NN_LB
                                + static_cast<std::size_t>(max_out) * dev::NN_LB + dev::NN_LB + 4u;
    const std::size_t bytes = doubles * sizeof(double);
    if (bytes + 2048u > smem_per_block_max) {
        return false;
    }
    allow_max_smem({hy::detail::nn_kernel_step(), hy::detail::nn_kernel_prop()}, smem_per_block_max);
    c.nnd = d;
    c.nn_wimg = std::move(img);
    const std::uint32_t grid = std::max(1u, std::min(n_sms, (n + dev::NN_LB - 1u) / dev::NN_LB));
    c.k = {kernel_sel::nn, 8, dev::NN_LB, 1, dev::NN_THREADS, 1u, grid, bytes, plan.n_slots};
    return true;
}

// The kernel a request selects (tape_mode as hy_batch_set_kernel() takes it, 0 automatic). A request that cannot run
// throws, and leaves the batch as it is.
candidate shard::decide(int want_mode, int L, int N, std::uint32_t threads, std::uint32_t blocks_per_sm) const
{
    candidate c;
    // Mode 8: the dense-network kernel (right-hand sides that are feed-forward networks, nn_plan.hpp); the automatic
    // mode takes it whenever the program qualifies.
    if (want_mode == 8 || (want_mode == 0 && opt_nn != 0)) {
        if (setup_nn(c)) {
            return c;
        }
        if (want_mode == 8) {
            throw std::invalid_argument("The dense-network kernel cannot run this program: "
                                        + (nnp.ok ? std::string("it does not fit in shared memory") : nnp.why));
        }
    }
    // Mode 6 / 7: the N-body kernel with warp / CTA teams.
    // Automatic mode takes it whenever the program qualifies (nb_plan.hpp).
    if (want_mode == 6 || want_mode == 7 || want_mode == 9 || (want_mode == 0 && opt_nb != 0)) {
        // Mode 9: one thread per lane (systems with one pair interaction); the automatic mode takes it when it applies,
        // an explicit mode 6 never does (it selects k_nb with the given team shape).
        const int lane = want_mode == 9 ? 1 : (want_mode == 0 ? (opt_nb1 != 0 ? -1 : 0) : 0);
        if (setup_nb(want_mode == 9 ? 32 : L, threads, want_mode == 0 ? -1 : (want_mode == 7 ? 1 : 0), lane, c)) {
            return c;
        }
        if (want_mode != 0) {
            throw std::invalid_argument("The N-body kernel cannot run this program: "
                                        + (nbp.ok ? std::string("no configuration fits on an SM") : nbp.why));
        }
    }
    if (want_mode == 4 || want_mode == 5) {
        setup_coop_global(L, N, threads, want_mode == 5 ? 1 : 0, c);
        return c;
    }
    if (want_mode == 1) {
        setup_hbm(threads, blocks_per_sm, c);
        return c;
    }
    if (want_mode == 3) {
        want_mode = 2;
    }
    if (setup_coop(L, N, threads, blocks_per_sm, c)) {
        return c;
    }
    if (want_mode == 2) {
        throw std::invalid_argument("The derivative tape of this system ("
                                    + std::to_string((c.tables ? c.tables->plan : plan).n_slots)
                                    + " doubles per lane) does not fit in shared memory");
    }
    // Automatic: the cooperative kernel with the tape in global memory.
    setup_coop_global(0, 0, 0, -1, c);
    return c;
}

// Installs a decided selection: releases the scratch of the current one, uploads the tables of the new one and
// allocates its scratch. Only CUDA errors can fail here.
void shard::commit(candidate c)
{
    const auto release = [](auto *&p) {
        if (p != nullptr) {
            HY_CUDA_CHECK(cudaFree(p));
            p = nullptr;
        }
    };
    release(d_gscratch);
    release(d_cscratch);
    release(d_nb_roles);
    release(d_nn_wimg);
    release(d_nn_out);
    if (c.tables) {
        set_tables(std::move(*c.tables));
    }
    d_gscratch = c.k.gscratch != 0u ? dalloc<double>(c.k.gscratch) : nullptr;
    d_cscratch = c.k.cscratch != 0u ? dalloc<double>(c.k.cscratch) : nullptr;
    if (c.k.family == kernel_sel::hbm) {
        h_threads = c.k.threads;
    } else if (c.k.family == kernel_sel::nb) {
        if (d_nb_pairs == nullptr) {
            d_nb_pairs = dupload(nbp.pairs);
            d_nb_consts = dupload(nbp.consts);
            d_nb_fac = dupload(nbp.fac);
        }
        d_nb_roles = dupload(c.nb_roles);
        nbd = c.nbd;
        nbd.pairs = d_nb_pairs;
        nbd.roles = reinterpret_cast<const uint4 *>(d_nb_roles);
        nbd.consts = d_nb_consts;
        nbd.fac = d_nb_fac;
        nbd.offchip = d_gscratch;
    } else if (c.k.family == kernel_sel::nn) {
        d_nn_wimg = dupload(c.nn_wimg);
        d_nn_out = dupload(nnp.out_of_sv);
        nnd = c.nnd;
        nnd.wimg = d_nn_wimg;
        nnd.out_of_sv = d_nn_out;
    }
    sel = c.k;
}

// The public Taylor-coefficient array, [n_eq][order + 1][batch] (src/taylor_00.cpp:574-580), is allocated the first
// time something needs it (write_tc, dense output, hy_batch_get_ptrs()): 6-body, 2^20 lanes: 6.3 GB; the
// cooperative kernels keep the coefficients of the current step in a private per-warp store otherwise.
void shard::ensure_tc()
{
    if (d_tc == nullptr) {
        // (With events, the rows of the event equations follow those of the state variables.)
        const std::size_t sz = static_cast<std::size_t>(n_eq + n_ev) * (order + 1u) * n;
        d_tc = dalloc<double>(sz);
        HY_CUDA_CHECK(cudaMemsetAsync(d_tc, 0, sizeof(double) * sz, stream));
    }
}

// ---- Event detection (ev_kernels.cuh) ----
// (The arguments are checked by hy_batch_set_events().)
void shard::ev_setup(std::uint32_t n_te, const std::int32_t *dirs, const double *cooldowns, double tol)
{
    for (void *q : ev_allocs) {
        HY_CUDA_CHECK(cudaFree(q));
    }
    ev_allocs.clear();
    const auto keep = [this](auto *q) {
        ev_allocs.push_back(static_cast<void *>(q));
        return q;
    };
    const std::uint32_t p = order, pp1 = p + 1u;
    dev::ev_args E{};
    E.n_ev = n_ev;
    E.n_te = n_te;
    E.tol = tol;
    E.max_svf = *std::max_element(prog_host->ev_defs.begin(), prog_host->ev_defs.end());
    E.ev_defs = keep(dupload(prog_host->ev_defs));
    E.dirs = keep(dupload(std::vector<int>(dirs, dirs + n_ev)));
    E.cooldowns = keep(dupload(std::vector<double>(cooldowns, cooldowns + n_te)));
    // Binomial coefficients, exact in double precision for the orders in use (src/detail/llvm_helpers_ed.cpp:421-455).
    std::vector<double> bc(static_cast<std::size_t>(pp1) * pp1, 0.);
    for (std::uint32_t i = 0; i <= p; ++i) {
        bc[i * pp1] = 1.;
        for (std::uint32_t j = 1; j <= i; ++j) {
            bc[i * pp1 + j] = bc[(i - 1u) * pp1 + j - 1u] + (j < i ? bc[(i - 1u) * pp1 + j] : 0.);
        }
    }
    E.bc = keep(dupload(bc));
    const std::size_t B = n;
    E.h = keep(dalloc<double>(B));
    E.mdt = keep(dalloc<double>(B));
    E.g_eps = keep(dalloc<double>(B));
    E.cd = keep(dalloc<double>(B * 2u * std::max(n_te, 1u)));
    E.cd_on = keep(dalloc<unsigned char>(B * std::max(n_te, 1u)));
    HY_CUDA_CHECK(cudaMemset(E.cd_on, 0, B * std::max(n_te, 1u)));
    // (Inactive cooldowns read back as zeros, not as whatever the allocation held.)
    HY_CUDA_CHECK(cudaMemset(E.cd, 0, sizeof(double) * B * 2u * std::max(n_te, 1u)));
    E.cand = keep(dalloc<std::uint32_t>(B * n_ev));
    E.counters = keep(dalloc<unsigned>(4));
    E.rec_cap = static_cast<std::uint32_t>(std::min<std::size_t>(std::max<std::size_t>(B * n_ev, 1024u), 1u << 26));
    E.rec = keep(dalloc<dev::ev_rec>(E.rec_cap));
    E.te_key = keep(dalloc<unsigned long long>(B));
    E.te_sel = keep(dalloc<unsigned long long>(B));
    // One bisection stack per detecting thread: a fraction of the lanes ever needs one at the same time.
    E.arena_threads = 64u * std::min<std::uint32_t>(n_sms, static_cast<std::uint32_t>((B * n_ev + 63u) / 64u));
    E.arena = keep(dalloc<double>(static_cast<std::size_t>(dev::EV_STACK) * (pp1 + 2u) * E.arena_threads));
    eva = E;
}

// One event step; returns the events found, in the order the callbacks must run.
std::vector<hy_event_rec> shard::ev_step(const double *d_mdt, int backward)
{
    if (sel.family != kernel_sel::hbm) {
        commit(decide(1, 0, 0, 0, 0));
    }
    ensure_tc();
    const std::uint32_t B = n;
    dev::run_args R{};
    R.max_delta_t = d_mdt;
    R.default_max_delta_t = backward ? -std::numeric_limits<double>::infinity() : std::numeric_limits<double>::infinity();
    R.counter = d_counter;
    R.flags = d_flags;
    HY_CUDA_CHECK(cudaMemsetAsync(d_counter, 0, sizeof(unsigned int), stream));
    dev::k_ev_jet<<<sel.grid, sel.threads, 0, stream>>>(prog, view(), R, eva, d_gscratch, slab_doubles);
    HY_CUDA_CHECK(cudaGetLastError());
    n_launches += 1;
    unsigned counters[4] = {0u, 0u, 0u, 0u};
    for (;;) {
        HY_CUDA_CHECK(cudaMemsetAsync(eva.counters, 0, 4u * sizeof(unsigned), stream));
        const std::size_t n_pairs = static_cast<std::size_t>(n_ev) * B;
        dev::k_ev_fex<<<static_cast<unsigned>((n_pairs + 255u) / 256u), 256, 0, stream>>>(prog, view(), eva);
        dev::k_ev_detect<<<eva.arena_threads / 64u, 64, 0, stream>>>(prog, view(), eva);
        HY_CUDA_CHECK(cudaGetLastError());
        n_launches += 2;
        HY_CUDA_CHECK(cudaMemcpyAsync(counters, eva.counters, sizeof(counters), cudaMemcpyDeviceToHost, stream));
        HY_CUDA_CHECK(cudaStreamSynchronize(stream));
        if (counters[1] <= eva.rec_cap) {
            break;
        }
        // More events than record slots (never seen in practice: one slot per (event, lane) pair): grow and redo the
        // detection, which only reads the jet.
        const std::uint32_t new_cap = counters[1] + counters[1] / 2u;
        dev::ev_rec *nr = dalloc<dev::ev_rec>(new_cap);
        for (auto &q : ev_allocs) {
            if (q == static_cast<void *>(eva.rec)) {
                q = nr;
            }
        }
        HY_CUDA_CHECK(cudaFree(eva.rec));
        eva.rec = nr;
        eva.rec_cap = new_cap;
        HY_CUDA_CHECK(cudaMemsetAsync(eva.te_key, 0xff, sizeof(unsigned long long) * B, stream));
    }
    const unsigned n_rec = counters[1];
    if (n_rec != 0u) {
        dev::k_ev_first<<<(n_rec + 127u) / 128u, 128, 0, stream>>>(view(), eva);
        ++n_launches;
    }
    dev::k_ev_apply<<<(B + 127u) / 128u, 128, 0, stream>>>(prog, view(), eva);
    ++n_launches;
    std::vector<hy_event_rec> evs;
    if (n_rec != 0u) {
        dev::k_ev_filter<<<(n_rec + 127u) / 128u, 128, 0, stream>>>(view(), eva);
        ++n_launches;
        std::vector<dev::ev_rec> recs(n_rec);
        HY_CUDA_CHECK(cudaMemcpyAsync(recs.data(), eva.rec, sizeof(dev::ev_rec) * n_rec, cudaMemcpyDeviceToHost, stream));
        HY_CUDA_CHECK(cudaStreamSynchronize(stream));
        for (const auto &r : recs) {
            if (r.live != 0u) {
                evs.push_back(hy_event_rec{r.lane, r.idx, r.terminal, r.d_sgn, r.t, r.abs_der});
            }
        }
        // Per lane: the non-terminal events in time order (src/taylor_adaptive_batch.cpp:789-790: by |t|; equal times
        // keep the order of the event indices), then the terminal event.
        std::sort(evs.begin(), evs.end(), [](const hy_event_rec &a, const hy_event_rec &b) {
            if (a.lane != b.lane) {
                return a.lane < b.lane;
            }
            if (a.terminal != b.terminal) {
                return a.terminal < b.terminal;
            }
            if (std::abs(a.t) != std::abs(b.t)) {
                return std::abs(a.t) < std::abs(b.t);
            }
            return a.idx < b.idx;
        });
    }
    HY_CUDA_CHECK(cudaGetLastError());
    return evs;
}

void shard::launch(bool prop, const dev::run_args &R)
{
    if (R.write_tc != 0) {
        ensure_tc();
    }
    HY_CUDA_CHECK(cudaMemsetAsync(d_counter, 0, sizeof(unsigned int), stream));
    const kernel_sel &k = sel;
    switch (k.family) {
    case kernel_sel::hbm:
        (prop ? dev::k_hbm<true> : dev::k_hbm<false>)<<<k.grid, k.threads, 0, stream>>>(prog, view(), R, d_gscratch,
                                                                                        slab_doubles);
        break;
    case kernel_sel::nn:
        (prop ? hy::detail::nn_kernel_prop() : hy::detail::nn_kernel_step())<<<k.grid, k.threads, k.smem, stream>>>(
            prog, nnd, view(), R);
        break;
    case kernel_sel::coop:
    case kernel_sel::nb: {
        // The coefficients of a step go to the private per-warp store, or to tc on request. k_nb1 always works on its
        // private store ([order][slot][32 lanes], velocities only) and publishes the coefficients to tc on request.
        dev::run_args R2 = R;
        const bool pub = R.write_tc != 0, priv = !pub || k.tape_mode == 9;
        const auto lanes = static_cast<unsigned long long>(k.L);
        R2.coef_pub = pub ? 1 : 0;
        R2.coef_base = priv ? d_cscratch : d_tc;
        R2.coef_warp_stride = priv ? static_cast<unsigned long long>(order + 1u) * n_eq * lanes : 0ull;
        R2.coef_stride_sv = pub ? static_cast<unsigned long long>(order + 1u) * n : lanes;
        R2.coef_stride_o = pub ? static_cast<unsigned long long>(n) : static_cast<unsigned long long>(n_eq) * lanes;
        if (k.family == kernel_sel::nb) {
            (prop ? k.nbv->prop : k.nbv->step)<<<k.grid, k.threads, k.smem, stream>>>(prog, nbd, view(), R2);
        } else {
            (prop ? k.cv->prop : k.cv->step)<<<k.grid, k.threads, k.smem, stream>>>(prog, d_blob, view(), R2,
                                                                                    d_gscratch);
        }
        break;
    }
    }
    HY_CUDA_CHECK(cudaGetLastError());
    ++n_launches;
}

// The rows the propagate entry points reduce (run_args::angles), or null. The N-body and dense-network kernels have no
// reduction (their programs hold no angles): a non-empty list is refused there.
const unsigned char *shard::prop_angles() const
{
    if (!angles_on) {
        return nullptr;
    }
    if (sel.family == kernel_sel::nb || sel.family == kernel_sel::nn) {
        throw hy::detail::not_implemented_error("The angle reducer runs on the device only in the cooperative and the "
                                                "HBM kernels, not in the N-body or dense-network kernel selected for "
                                                "this batch");
    }
    return d_angles;
}

namespace
{

struct device_guard {
    int prev = 0;
    explicit device_guard(int dev)
    {
        HY_CUDA_CHECK(cudaGetDevice(&prev));
        if (prev != dev) {
            HY_CUDA_CHECK(cudaSetDevice(dev));
        }
    }
    ~device_guard()
    {
        cudaSetDevice(prev);
    }
};

// Device memory freed when its owner goes.
struct cuda_free {
    void operator()(void *p) const noexcept
    {
        cudaFree(p);
    }
};
template <typename T>
using dev_ptr = std::unique_ptr<T, cuda_free>;

template <typename T>
dev_ptr<T> dev_alloc(std::size_t count)
{
    void *p = nullptr;
    HY_CUDA_CHECK(cudaMalloc(&p, sizeof(T) * count));
    return dev_ptr<T>(static_cast<T *>(p));
}

// The device state of `lanes` lanes of the program on `device`.
std::unique_ptr<shard> make_shard(const hy_program &p, std::uint32_t lanes, int device)
{
    // Overflow checks on the buffer sizes, like src/taylor_adaptive_batch.cpp:256-264,375-378.
    const std::uint64_t tc_size = static_cast<std::uint64_t>(p.n_eq) * (p.order + 1u) * lanes;
    if (tc_size > (std::numeric_limits<std::uint64_t>::max() >> 4)) {
        throw std::overflow_error("Overflow detected while computing the size of the Taylor coefficients buffer");
    }

    auto sh = std::make_unique<shard>();
    sh->device = device;
    device_guard guard(device);

    sh->n = lanes;
    sh->n_eq = p.n_eq;
    sh->n_pars = p.n_pars;
    sh->order = p.order;
    sh->n_uvars = p.n_uvars;
    sh->high_accuracy = p.high_accuracy;

    cudaDeviceProp prop{};
    HY_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
    sh->n_sms = static_cast<std::uint32_t>(prop.multiProcessorCount);
    sh->smem_per_block_max = prop.sharedMemPerBlockOptin;
    sh->smem_per_sm = prop.sharedMemPerMultiprocessor;

    // Program arrays, "hbm" encoding.
    static_assert(sizeof(hy_op) == sizeof(uint4), "hy_op must be 16 bytes");
    sh->d_ops = reinterpret_cast<uint4 *>(sh->dupload(p.ops));
    sh->d_args = sh->dupload(p.args);
    sh->d_consts = sh->dupload(p.consts);
    sh->d_sv_defs = sh->dupload(p.sv_defs);

    auto &P = sh->prog;
    P.n_eq = p.n_eq;
    P.n_uvars = p.n_uvars;
    P.n_pars = p.n_pars;
    P.order = p.order;
    P.n_ops = p.n_uvars - p.n_eq;
    P.high_accuracy = p.high_accuracy ? 1 : 0;
    // taylor_determine_h_rhofac(), src/taylor_00.cpp:84-94 (host libm, like the reference's number arithmetic).
    P.rhofac = std::exp((-7. / 10.) / static_cast<double>(p.order - 1u)) / (std::exp(1.) * std::exp(1.));
    P.inv_p = 1. / static_cast<double>(p.order);
    P.inv_pm1 = 1. / static_cast<double>(p.order - 1u);
    P.ops = sh->d_ops;
    P.args = sh->d_args;
    P.consts = sh->d_consts;
    P.sv_defs = sh->d_sv_defs;

    // Cooperative plan.
    // HEYOKA_B200_FUSE=0 disables the superinstructions, HEYOKA_B200_FUSE_SV=0 the fused state-variable
    // propagation, HEYOKA_B200_SPILL=0/1 forces the overflow tape off/on (diagnostics / tests).
    if (const char *env = std::getenv("HEYOKA_B200_FUSE")) {
        sh->opt_fuse = std::string{env} != "0";
    }
    if (const char *env = std::getenv("HEYOKA_B200_FUSE_SV")) {
        sh->opt_fuse_sv = std::string{env} != "0";
    }
    if (const char *env = std::getenv("HEYOKA_B200_SPILL")) {
        sh->opt_spill = std::string{env} != "0" ? 1 : 0;
    }
    if (const char *env = std::getenv("HEYOKA_B200_NB")) {
        sh->opt_nb = std::string{env} != "0" ? 1 : 0;
    }
    if (const char *env = std::getenv("HEYOKA_B200_NB_LANE")) {
        sh->opt_nb1 = std::string{env} != "0" ? 1 : 0;
    }
    if (const char *env = std::getenv("HEYOKA_B200_NB_THREADS")) {
        sh->opt_nb_threads = static_cast<std::uint32_t>(std::atoi(env));
    }
    sh->prog_host = std::make_shared<const hy_program>(p);
    sh->set_tables(sh->make_tables(false));
    sh->slab_doubles = static_cast<std::size_t>(p.n_uvars) * (p.order + 1u) * 32u;
    sh->nbp = hy::detail::make_nb_plan(p);
    if (const char *env = std::getenv("HEYOKA_B200_NN")) {
        sh->opt_nn = std::string{env} != "0" ? 1 : 0;
    }
    sh->nnp = hy::detail::make_nn_plan(p);

    // Resident arrays.
    const std::size_t n = lanes;
    sh->d_state = sh->dalloc<double>(n * p.n_eq);
    sh->d_pars = sh->dalloc<double>(n * p.n_pars);
    sh->d_t_hi = sh->dalloc<double>(n);
    sh->d_t_lo = sh->dalloc<double>(n);
    sh->d_last_h = sh->dalloc<double>(n);
    sh->d_d_out = sh->dalloc<double>(n * p.n_eq);
    sh->d_step_outcome = sh->dalloc<long long>(n);
    sh->d_prop_outcome = sh->dalloc<long long>(n);
    sh->d_prop_min_h = sh->dalloc<double>(n);
    sh->d_prop_max_h = sh->dalloc<double>(n);
    sh->d_prop_n_steps = sh->dalloc<unsigned long long>(n);
    sh->d_prop_iters = sh->dalloc<unsigned long long>(n);
    sh->d_skip = sh->dalloc<unsigned char>(n);
    sh->d_tmp = sh->dalloc<double>(3u * n);
    sh->d_snapshot = sh->dalloc<double>(n * (p.n_eq + 2u));
    sh->d_counter = sh->dalloc<unsigned int>(1);
    sh->d_flags = sh->dalloc<dev::run_flags>(2); // (+ scratch words behind the flags)

    HY_CUDA_CHECK(cudaMemset(sh->d_state, 0, sizeof(double) * n * p.n_eq));
    HY_CUDA_CHECK(cudaMemset(sh->d_pars, 0, sizeof(double) * std::max<std::size_t>(n * p.n_pars, 1u)));
    HY_CUDA_CHECK(cudaMemset(sh->d_t_hi, 0, sizeof(double) * n));
    HY_CUDA_CHECK(cudaMemset(sh->d_t_lo, 0, sizeof(double) * n));
    HY_CUDA_CHECK(cudaMemset(sh->d_last_h, 0, sizeof(double) * n));

    // Kernel selection: HEYOKA_B200_TAPE = hbm | smem overrides the automatic choice.
    int want = 0;
    if (const char *env = std::getenv("HEYOKA_B200_TAPE")) {
        const std::string s{env};
        want = s == "hbm" ? 1 : (s == "smem" ? 2 : 0);
    }
    sh->n_ev = static_cast<std::uint32_t>(p.ev_defs.size());
    if (sh->n_ev != 0u) {
        // Event detection runs on the thread-per-lane kernel family (ev_kernels.cuh).
        if (p.order + 1u > static_cast<std::uint32_t>(dev::EV_MAXP1)) {
            throw hy::detail::not_implemented_error("Event detection supports Taylor orders up to "
                                                    + std::to_string(dev::EV_MAXP1 - 1));
        }
        want = 1;
    }
    sh->commit(sh->decide(want, 0, 0, 0, 0));
    return sh;
}

// A batch of `batch` lanes in contiguous blocks, as even as possible, one per entry of devs (< 0: the current device);
// never more shards than lanes.
std::unique_ptr<hy_batch> make_batch(const hy_program &p, std::uint32_t batch, const std::vector<int> &devs, int n_dev,
                                     bool multi)
{
    auto b = std::make_unique<hy_batch>();
    b->n = batch;
    b->n_eq = p.n_eq;
    b->n_ev = static_cast<std::uint32_t>(p.ev_defs.size());
    b->multi = multi;
    const std::uint32_t ns = std::min<std::uint32_t>(static_cast<std::uint32_t>(devs.size()), batch);
    b->off.push_back(0u);
    for (std::uint32_t i = 0; i < ns; ++i) {
        int device = devs[i];
        if (device < 0) {
            HY_CUDA_CHECK(cudaGetDevice(&device));
        }
        if (device >= n_dev) {
            throw std::invalid_argument("Invalid CUDA device index " + std::to_string(device));
        }
        const std::uint32_t lanes = batch / ns + (i < batch % ns ? 1u : 0u);
        b->shards.push_back(make_shard(p, lanes, device));
        b->off.push_back(b->off.back() + lanes);
    }
    return b;
}

// ------------------------------------------------------------------------------------------------
// Every entry point runs on the shards of its batch: the lanes are independent ODE systems, so a batch shards over the
// GPUs of a box with no data-path communication (src/ensemble_propagate.cpp:192-311 partitions its members over TBB
// threads the same way). The only coupling is the reference's GLOBAL exits of propagate_until() (non-finite state
// anywhere, iteration limit, length of the lock-step loop), applied across the shards between the phases of
// propagate().
// ------------------------------------------------------------------------------------------------

// fn(shard, i) on every shard, under the shard's device. One shard: on the calling thread. More: one host thread per
// shard, so that the shards' copies and kernels overlap. The first failure in shard order is rethrown as it was thrown.
template <typename F>
void for_each_shard(hy_batch *b, F &&fn)
{
    const std::size_t ns = b->shards.size();
    if (ns == 1u) {
        device_guard guard(b->shards[0]->device);
        fn(*b->shards[0], std::size_t(0));
        return;
    }
    std::vector<std::exception_ptr> errs(ns);
    std::vector<std::thread> thr;
    thr.reserve(ns);
    for (std::size_t i = 0; i < ns; ++i) {
        thr.emplace_back([&, i] {
            try {
                shard &sh = *b->shards[i];
                device_guard guard(sh.device);
                fn(sh, i);
            } catch (...) {
                errs[i] = std::current_exception();
            }
        });
    }
    for (auto &t : thr) {
        t.join();
    }
    for (const auto &e : errs) {
        if (e) {
            std::rethrow_exception(e);
        }
    }
}

// rows x (shard lanes) block of a host array with `pitch` elements per row, starting at column `off`. (The shard of an
// unsharded batch takes the same pitched copy, with pitch = width: no slower than a flat copy on an H100.)
template <typename T>
void rows_h2d(shard &sh, T *dst, const T *src, std::size_t rows, std::size_t pitch, std::size_t off)
{
    if (src != nullptr && rows != 0u) {
        HY_CUDA_CHECK(cudaMemcpy2DAsync(dst, sizeof(T) * sh.n, src + off, sizeof(T) * pitch, sizeof(T) * sh.n, rows,
                                        cudaMemcpyHostToDevice, sh.stream));
    }
}
template <typename T>
void rows_d2h(shard &sh, T *dst, const T *src, std::size_t rows, std::size_t pitch, std::size_t off)
{
    if (dst != nullptr && rows != 0u) {
        HY_CUDA_CHECK(cudaMemcpy2DAsync(dst + off, sizeof(T) * pitch, src, sizeof(T) * sh.n, sizeof(T) * sh.n, rows,
                                        cudaMemcpyDeviceToHost, sh.stream));
    }
}

// The shard's lanes [off, off + n) of a per-lane array: a host array is staged into slot `slot` of d_tmp, a device
// array (on_device, an unsharded batch's) is used in place.
const double *stage(shard &sh, const double *src, int on_device, std::size_t off, std::uint32_t slot)
{
    if (src == nullptr || on_device) {
        return src;
    }
    double *dst = sh.d_tmp + static_cast<std::size_t>(slot) * sh.n;
    HY_CUDA_CHECK(cudaMemcpyAsync(dst, src + off, sizeof(double) * sh.n, cudaMemcpyHostToDevice, sh.stream));
    return dst;
}

void download(hy_batch *b, double *state, double *t_hi, double *t_lo, double *last_h)
{
    for_each_shard(b, [&](shard &sh, std::size_t i) {
        rows_d2h(sh, state, sh.d_state, sh.n_eq, b->n, b->off[i]);
        rows_d2h(sh, t_hi, sh.d_t_hi, 1u, b->n, b->off[i]);
        rows_d2h(sh, t_lo, sh.d_t_lo, 1u, b->n, b->off[i]);
        rows_d2h(sh, last_h, sh.d_last_h, 1u, b->n, b->off[i]);
        HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
    });
}

// propagate_until() on one shard, in three phases so that the reference's GLOBAL exits apply across the shards:
//   phase 1  snapshot of (state, time), one launch of the propagate kernel, flags read back (synchronises);
//   replay   if a lane of ANY shard went non-finite: restore the snapshot and re-run with the iteration count capped at
//            the first such iteration (the reference stops EVERY lane there, src/taylor_adaptive_batch.cpp:1462-1467;
//            lanes are independent, so the capped re-run reproduces it exactly);
//   finish   iteration limit -> every lane reports step_limit (:1516-1526); the lanes that were done before the loop's
//            last iteration K took zero-length steps in the reference: last_h = 0 and, with write_tc, Taylor
//            coefficients re-expanded about the final state (one masked zero-length step).
struct prop_ctx {
    dev::run_args R{};
    dev::run_flags fl{};
};

void propagate_phase1(shard &sh, const double *d_tf_hi, const double *d_tf_lo, const double *d_mdt, uint64_t max_steps,
                      int write_tc, const unsigned char *angles, prop_ctx &c)
{
    const std::size_t state_doubles = static_cast<std::size_t>(sh.n_eq) * sh.n;
    HY_CUDA_CHECK(cudaMemcpyAsync(sh.d_snapshot, sh.d_state, sizeof(double) * state_doubles, cudaMemcpyDeviceToDevice,
                                  sh.stream));
    HY_CUDA_CHECK(cudaMemcpyAsync(sh.d_snapshot + state_doubles, sh.d_t_hi, sizeof(double) * sh.n,
                                  cudaMemcpyDeviceToDevice, sh.stream));
    HY_CUDA_CHECK(cudaMemcpyAsync(sh.d_snapshot + state_doubles + sh.n, sh.d_t_lo, sizeof(double) * sh.n,
                                  cudaMemcpyDeviceToDevice, sh.stream));
    const dev::run_flags init{0u, 0u, ~0ull, 0ull};
    HY_CUDA_CHECK(cudaMemcpyAsync(sh.d_flags, &init, sizeof(init), cudaMemcpyHostToDevice, sh.stream));
    c.R = dev::run_args{};
    c.R.max_delta_t = d_mdt;
    c.R.tf_hi = d_tf_hi;
    c.R.tf_lo = d_tf_lo;
    c.R.iter_cap = max_steps;
    c.R.replay = 0;
    c.R.write_tc = write_tc;
    c.R.flags = sh.d_flags;
    c.R.counter = sh.d_counter;
    c.R.angles = angles;
    sh.launch(true, c.R);
    HY_CUDA_CHECK(cudaMemcpyAsync(&c.fl, sh.d_flags, sizeof(c.fl), cudaMemcpyDeviceToHost, sh.stream));
    HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
}

void propagate_replay(shard &sh, prop_ctx &c, unsigned long long cap)
{
    const std::size_t state_doubles = static_cast<std::size_t>(sh.n_eq) * sh.n;
    HY_CUDA_CHECK(cudaMemcpyAsync(sh.d_state, sh.d_snapshot, sizeof(double) * state_doubles, cudaMemcpyDeviceToDevice,
                                  sh.stream));
    HY_CUDA_CHECK(cudaMemcpyAsync(sh.d_t_hi, sh.d_snapshot + state_doubles, sizeof(double) * sh.n,
                                  cudaMemcpyDeviceToDevice, sh.stream));
    HY_CUDA_CHECK(cudaMemcpyAsync(sh.d_t_lo, sh.d_snapshot + state_doubles + sh.n, sizeof(double) * sh.n,
                                  cudaMemcpyDeviceToDevice, sh.stream));
    const dev::run_flags init{0u, 0u, ~0ull, 0ull};
    HY_CUDA_CHECK(cudaMemcpyAsync(sh.d_flags, &init, sizeof(init), cudaMemcpyHostToDevice, sh.stream));
    c.R.iter_cap = cap;
    c.R.replay = 1;
    sh.launch(true, c.R);
    HY_CUDA_CHECK(cudaMemcpyAsync(&c.fl, sh.d_flags, sizeof(c.fl), cudaMemcpyDeviceToHost, sh.stream));
    HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
}

// ex: the flags of the whole batch (any_nf from phase 1, any_limit and max_iter from the last launch).
// (With the angle reducer there is nothing to reduce here: every lane takes at least the first iteration of the
// kernel's loop, a zero-length step for a lane already at its final time, and that step reduces it.)
void propagate_finish(shard &sh, const dev::run_flags &ex, int write_tc)
{
    const std::uint32_t gb = (sh.n + 255u) / 256u;
    if (ex.any_nf == 0u && ex.any_limit != 0u) {
        dev::k_fill_outcome<<<gb, 256, 0, sh.stream>>>(sh.d_prop_outcome, sh.n, HY_OUTCOME_STEP_LIMIT);
        HY_CUDA_CHECK(cudaGetLastError());
        ++sh.n_launches;
    }
    // Lanes that were done before the last iteration of the reference's loop.
    unsigned *d_any = reinterpret_cast<unsigned *>(sh.d_flags) + sizeof(dev::run_flags) / sizeof(unsigned);
    HY_CUDA_CHECK(cudaMemsetAsync(d_any, 0, sizeof(unsigned), sh.stream));
    dev::k_prop_early<<<gb, 256, 0, sh.stream>>>(sh.d_prop_iters, ex.max_iter, sh.n, sh.d_last_h, sh.d_skip, sh.d_tmp,
                                                 d_any);
    HY_CUDA_CHECK(cudaGetLastError());
    ++sh.n_launches;
    if (write_tc != 0) {
        unsigned any = 0;
        HY_CUDA_CHECK(cudaMemcpyAsync(&any, d_any, sizeof(any), cudaMemcpyDeviceToHost, sh.stream));
        HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        if (any != 0u) {
            dev::run_args R{};
            R.max_delta_t = sh.d_tmp; // zeros
            R.write_tc = 1;
            R.flags = sh.d_flags;
            R.counter = sh.d_counter;
            R.skip = sh.d_skip;
            sh.launch(false, R);
        }
    }
}

// The host arrays of hy_batch_propagate_until_host() (NULL: not wanted).
struct prop_host {
    const double *state_in, *pars, *t_hi_in, *t_lo_in;
    double *state, *t_hi, *t_lo, *last_h;
    int64_t *outcome;
    double *min_h, *max_h;
    uint64_t *n_steps;
};

void download_prop(shard &sh, const prop_host &h, std::size_t pitch, std::size_t off)
{
    rows_d2h(sh, h.state, sh.d_state, sh.n_eq, pitch, off);
    rows_d2h(sh, h.t_hi, sh.d_t_hi, 1u, pitch, off);
    rows_d2h(sh, h.t_lo, sh.d_t_lo, 1u, pitch, off);
    rows_d2h(sh, reinterpret_cast<long long *>(h.outcome), sh.d_prop_outcome, 1u, pitch, off);
    rows_d2h(sh, h.min_h, sh.d_prop_min_h, 1u, pitch, off);
    rows_d2h(sh, h.max_h, sh.d_prop_max_h, 1u, pitch, off);
    rows_d2h(sh, reinterpret_cast<unsigned long long *>(h.n_steps), sh.d_prop_n_steps, 1u, pitch, off);
}

// propagate_until() of every lane of the batch to per-lane final times (host arrays, or device arrays of an unsharded
// batch: on_device). With io, the shard's slice of the state and times is uploaded before and its results downloaded
// after its own kernel: the state right away, last_h (and the outcomes, if the iteration limit was hit) once the global
// exits are known. Returns the flags of the whole batch.
// With reduce, the angle reducer of hy_batch_set_angles() runs after every step.
dev::run_flags propagate(hy_batch *b, const double *tf_hi, const double *tf_lo, const double *mdt, int on_device,
                         uint64_t max_steps, int write_tc, const prop_host *io, bool reduce = true)
{
    std::vector<prop_ctx> ctx(b->shards.size());
    std::vector<const unsigned char *> angles(b->shards.size());
    for (std::size_t i = 0; i < b->shards.size(); ++i) {
        angles[i] = reduce ? b->shards[i]->prop_angles() : nullptr;
    }
    for_each_shard(b, [&](shard &sh, std::size_t i) {
        const std::size_t off = b->off[i];
        if (io != nullptr) {
            rows_h2d(sh, sh.d_state, io->state_in, sh.n_eq, b->n, off);
            rows_h2d(sh, sh.d_pars, io->pars, sh.n_pars, b->n, off);
            rows_h2d(sh, sh.d_t_hi, io->t_hi_in, 1u, b->n, off);
            rows_h2d(sh, sh.d_t_lo, io->t_lo_in, 1u, b->n, off);
        }
        propagate_phase1(sh, stage(sh, tf_hi, on_device, off, 0), stage(sh, tf_lo, on_device, off, 1),
                         stage(sh, mdt, on_device, off, 2), max_steps, write_tc, angles[i], ctx[i]);
        if (io != nullptr) {
            download_prop(sh, *io, b->n, off); // (speculative: a non-finite lane anywhere makes every shard run again)
        }
    });
    dev::run_flags ex{0u, 0u, ~0ull, 0ull};
    for (const auto &c : ctx) {
        if (c.fl.any_nf != 0u) {
            ex.any_nf = 1u;
            ex.min_nf_iter = std::min(ex.min_nf_iter, c.fl.min_nf_iter);
        }
    }
    if (ex.any_nf != 0u) {
        // Every lane of every shard stops at the first iteration in which any lane went non-finite.
        for_each_shard(b, [&](shard &sh, std::size_t i) { propagate_replay(sh, ctx[i], ex.min_nf_iter); });
    }
    for (const auto &c : ctx) {
        ex.any_limit = ex.any_limit != 0u || c.fl.any_limit != 0u ? 1u : 0u;
        ex.max_iter = std::max(ex.max_iter, c.fl.max_iter);
    }
    for_each_shard(b, [&](shard &sh, std::size_t i) {
        propagate_finish(sh, ex, write_tc);
        if (io != nullptr) {
            if (ex.any_nf != 0u || ex.any_limit != 0u) {
                download_prop(sh, *io, b->n, b->off[i]);
            }
            rows_d2h(sh, io->last_h, sh.d_last_h, 1u, b->n, b->off[i]);
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        }
    });
    return ex;
}

// The device-resident propagations refuse a batch with event equations.
void refuse_events(const hy_batch *b)
{
    if (b != nullptr && b->n_ev != 0u) {
        throw hy::detail::not_implemented_error("A batch with event equations is propagated by the front end's lock-step "
                                                "loop over hy_batch_step(), not by the device-resident propagation");
    }
}

// The checks of propagate_until_impl() that need the CURRENT times (src/taylor_adaptive_batch.cpp:1212-1273): finite,
// and final time - current time representable (check_prop_times(): 16 bytes per lane come back from the device for them).
void check_prop_times_host(std::uint32_t n, const double *t_hi, const double *t_lo, const double *tf_hi, const double *tf_lo)
{
    for (std::uint32_t i = 0; i < n; ++i) {
        if (!std::isfinite(t_hi[i]) || !std::isfinite(t_lo[i])) {
            throw std::invalid_argument("Cannot invoke the propagate_until() function of an adaptive Taylor integrator "
                                        "in batch mode if one of the current times is not finite");
        }
    }
    for (std::uint32_t i = 0; i < n; ++i) {
        // (Same arithmetic as the device: Knuth two-sum of the high parts is enough to detect the overflow.)
        const double rem = tf_hi[i] - t_hi[i] + ((tf_lo != nullptr ? tf_lo[i] : 0.) - t_lo[i]);
        if (!std::isfinite(rem)) {
            throw std::invalid_argument("The final time passed to the propagate_until() function of an adaptive Taylor "
                                        "integrator in batch mode results in an overflow condition");
        }
    }
}

void check_prop_times(hy_batch *b, const double *tf_hi, const double *tf_lo)
{
    std::vector<double> t_hi(b->n), t_lo(b->n);
    download(b, nullptr, t_hi.data(), t_lo.data(), nullptr);
    check_prop_times_host(b->n, t_hi.data(), t_lo.data(), tf_hi, tf_lo);
}

// Argument checks of propagate_until_impl(), src/taylor_adaptive_batch.cpp:1212-1241.
void check_prop_args(std::uint32_t n, const double *t_final_hi, const double *t_final_lo, const double *max_delta_t)
{
    for (std::uint32_t i = 0; i < n; ++i) {
        if (!std::isfinite(t_final_hi[i]) || (t_final_lo != nullptr && !std::isfinite(t_final_lo[i]))) {
            throw std::invalid_argument("A non-finite time was passed to the propagate_until() function of an "
                                        "adaptive Taylor integrator in batch mode");
        }
        if (max_delta_t != nullptr) {
            if (std::isnan(max_delta_t[i])) {
                throw std::invalid_argument("A nan max_delta_t was passed to the propagate_until() function of an "
                                            "adaptive Taylor integrator in batch mode");
            }
            if (max_delta_t[i] <= 0) {
                throw std::invalid_argument("A non-positive max_delta_t was passed to the propagate_until() "
                                            "function of an adaptive Taylor integrator in batch mode");
            }
        }
    }
}

} // namespace

extern "C" {

int hy_batch_create(const hy_program *p, uint32_t batch, int device, hy_batch **out)
{
    try {
        if (p == nullptr || out == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_batch_create()");
        }
        if (batch == 0u) {
            throw std::invalid_argument("The batch size in an adaptive Taylor integrator cannot be zero");
        }
        int n_dev = 0;
        if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
            throw cuda_error("No usable CUDA device: heyoka_b200 has no CPU fallback");
        }
        *out = make_batch(*p, batch, {device}, n_dev, false).release();
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_create_multi(const hy_program *p, uint32_t batch, const int *devices, uint32_t n_devices, hy_batch **out)
{
    try {
        if (p == nullptr || out == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_batch_create_multi()");
        }
        int n_dev = 0;
        if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
            throw cuda_error("No usable CUDA device: heyoka_b200 has no CPU fallback");
        }
        std::vector<int> devs;
        if (devices == nullptr || n_devices == 0u) {
            for (int d = 0; d < n_dev; ++d) {
                devs.push_back(d);
            }
        } else {
            devs.assign(devices, devices + n_devices);
        }
        if (batch == 0u) {
            throw std::invalid_argument("The batch size in an adaptive Taylor integrator cannot be zero");
        }
        *out = make_batch(*p, batch, devs, n_dev, true).release();
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_device_count(void)
{
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess) {
        return 0;
    }
    return n_dev;
}

uint32_t hy_batch_n_shards(const hy_batch *b)
{
    return b == nullptr || !b->multi ? 0u : static_cast<uint32_t>(b->shards.size());
}

void hy_batch_destroy(hy_batch *b)
{
    delete b;
}

int hy_selftest_div(uint64_t n, uint64_t seed, uint64_t *mismatches)
{
    try {
        if (mismatches == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_selftest_div()");
        }
        unsigned long long *d = nullptr;
        HY_CUDA_CHECK(cudaMalloc(&d, sizeof(unsigned long long)));
        HY_CUDA_CHECK(cudaMemset(d, 0, sizeof(unsigned long long)));
        int dev_id = 0, n_sms = 0;
        HY_CUDA_CHECK(cudaGetDevice(&dev_id));
        HY_CUDA_CHECK(cudaDeviceGetAttribute(&n_sms, cudaDevAttrMultiProcessorCount, dev_id));
        dev::k_selftest_div<<<n_sms * 8, 256>>>(n, seed, d);
        HY_CUDA_CHECK(cudaGetLastError());
        unsigned long long h = 0;
        HY_CUDA_CHECK(cudaMemcpy(&h, d, sizeof(h), cudaMemcpyDeviceToHost));
        HY_CUDA_CHECK(cudaFree(d));
        *mismatches = h;
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_host_pin(void *ptr, size_t bytes)
{
    if (ptr == nullptr || bytes == 0u) {
        return HY_OK;
    }
    if (cudaHostRegister(ptr, bytes, cudaHostRegisterDefault) != cudaSuccess) {
        cudaGetLastError(); // (not fatal: the copies then go through the driver's staging buffers)
        hy::detail::set_last_error("cudaHostRegister() failed");
        return HY_ERR_CUDA;
    }
    return HY_OK;
}

int hy_host_unpin(void *ptr)
{
    if (ptr != nullptr && cudaHostUnregister(ptr) != cudaSuccess) {
        cudaGetLastError();
        return HY_ERR_CUDA;
    }
    return HY_OK;
}

int hy_batch_set_stream(hy_batch *b, void *cuda_stream)
{
    if (b != nullptr && b->multi) {
        hy::detail::set_last_error("hy_batch_set_stream() is not available on a multi-device batch");
        return HY_ERR_INVALID_ARG;
    }
    if (b == nullptr) {
        hy::detail::set_last_error("Null batch");
        return HY_ERR_INVALID_ARG;
    }
    b->shards[0]->stream = static_cast<cudaStream_t>(cuda_stream);
    return HY_OK;
}

int hy_batch_sync(hy_batch *b)
{
    try {
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        for_each_shard(b, [](shard &sh, std::size_t) { HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream)); });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_set_launch_config(hy_batch *b, uint32_t block_threads, uint32_t blocks_per_sm)
{
    try {
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        // Shard after shard, in shard order: shards on the same device size their scratch from the device memory the
        // previous shard left free (free_bytes_after_release()).
        for (auto &sh : b->shards) {
            device_guard guard(sh->device);
            HY_CUDA_CHECK(cudaStreamSynchronize(sh->stream));
            // The same tape mode and lanes (the N-body kernels derive their lanes per thread from the team; the network
            // kernel has a fixed shape and ignores every argument).
            const kernel_sel &k = sh->sel;
            sh->commit(sh->decide(k.tape_mode, k.L, k.family == kernel_sel::nb ? 0 : k.N, block_threads, blocks_per_sm));
        }
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_set_kernel(hy_batch *b, int tape_mode, uint32_t lanes_per_warp, uint32_t lanes_per_thread,
                        uint32_t block_threads, uint32_t blocks_per_sm)
{
    try {
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        if (tape_mode < 0 || tape_mode > 9) {
            throw std::invalid_argument("Invalid tape mode");
        }
        // (Shard after shard, in shard order, like hy_batch_set_launch_config().)
        for (auto &sh : b->shards) {
            device_guard guard(sh->device);
            HY_CUDA_CHECK(cudaStreamSynchronize(sh->stream));
            sh->commit(sh->decide(tape_mode, static_cast<int>(lanes_per_warp), static_cast<int>(lanes_per_thread),
                                  block_threads, blocks_per_sm));
        }
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_get_kernel(const hy_batch *b, hy_kernel_info *out)
{
    if (b == nullptr || out == nullptr) {
        hy::detail::set_last_error("Null pointer passed to hy_batch_get_kernel()");
        return HY_ERR_INVALID_ARG;
    }
    const shard &sh = *b->shards[0]; // (every shard runs the same kernel shape)
    const kernel_sel &k = sh.sel;
    out->tape_mode = k.tape_mode;
    out->lanes_per_warp = static_cast<uint32_t>(k.L);
    out->lanes_per_thread = static_cast<uint32_t>(k.N);
    out->block_threads = k.threads;
    out->blocks_per_sm = k.per_sm;
    out->grid = k.grid;
    out->smem_bytes = k.smem;
    out->tape_slots_per_lane = k.tape_slots;
    out->n_segments = sh.plan.n_segments;
    out->n_fused = sh.plan.n_fused;
    out->n_sms = sh.n_sms;
    out->tmem_cols_per_warp = 0u; // (sm_90 has no tensor memory)
    out->reserved = 0u;
    return HY_OK;
}

int hy_batch_set_angles(hy_batch *b, const uint32_t *sv_idx, uint32_t n)
{
    try {
        if (b == nullptr || (n != 0u && sv_idx == nullptr)) {
            throw std::invalid_argument("Null pointer passed to hy_batch_set_angles()");
        }
        std::vector<unsigned char> mask(b->n_eq, 0u);
        for (uint32_t k = 0; k < n; ++k) {
            if (sv_idx[k] >= b->n_eq) {
                throw std::invalid_argument("Invalid state variable index " + std::to_string(sv_idx[k])
                                            + " passed to hy_batch_set_angles(): the system has "
                                            + std::to_string(b->n_eq) + " state variables");
            }
            if (mask[sv_idx[k]] != 0u) {
                throw std::invalid_argument("The state variable index " + std::to_string(sv_idx[k])
                                            + " was passed twice to hy_batch_set_angles()");
            }
            mask[sv_idx[k]] = 1u;
        }
        for (auto &sh : b->shards) {
            sh->angles_on = n != 0u;
            if (n == 0u) {
                continue;
            }
            device_guard guard(sh->device);
            if (sh->d_angles == nullptr) {
                sh->d_angles = sh->dalloc<unsigned char>(b->n_eq);
            }
            // (Ordered on the shard's stream after the launches that read the previous list.)
            sh->angles = mask;
            HY_CUDA_CHECK(cudaMemcpyAsync(sh->d_angles, sh->angles.data(), sh->angles.size(), cudaMemcpyHostToDevice,
                                          sh->stream));
        }
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_upload(hy_batch *b, const double *state, const double *pars, const double *t_hi, const double *t_lo)
{
    try {
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            rows_h2d(sh, sh.d_state, state, sh.n_eq, b->n, b->off[i]);
            rows_h2d(sh, sh.d_pars, pars, sh.n_pars, b->n, b->off[i]);
            rows_h2d(sh, sh.d_t_hi, t_hi, 1u, b->n, b->off[i]);
            rows_h2d(sh, sh.d_t_lo, t_lo, 1u, b->n, b->off[i]);
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_download(hy_batch *b, double *state, double *t_hi, double *t_lo, double *last_h)
{
    try {
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        download(b, state, t_hi, t_lo, last_h);
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_download_step_res(hy_batch *b, int64_t *outcome, double *h)
{
    try {
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            rows_d2h(sh, reinterpret_cast<long long *>(outcome), sh.d_step_outcome, 1u, b->n, b->off[i]);
            rows_d2h(sh, h, sh.d_last_h, 1u, b->n, b->off[i]);
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_download_prop_res(hy_batch *b, int64_t *outcome, double *min_h, double *max_h, uint64_t *n_steps)
{
    try {
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            rows_d2h(sh, reinterpret_cast<long long *>(outcome), sh.d_prop_outcome, 1u, b->n, b->off[i]);
            rows_d2h(sh, min_h, sh.d_prop_min_h, 1u, b->n, b->off[i]);
            rows_d2h(sh, max_h, sh.d_prop_max_h, 1u, b->n, b->off[i]);
            rows_d2h(sh, reinterpret_cast<unsigned long long *>(n_steps), sh.d_prop_n_steps, 1u, b->n, b->off[i]);
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_download_tc(hy_batch *b, double *tc)
{
    try {
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            sh.ensure_tc();
            rows_d2h(sh, tc, sh.d_tc, static_cast<std::size_t>(sh.n_eq) * (sh.order + 1u), b->n, b->off[i]);
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_upload_tc(hy_batch *b, const double *tc)
{
    try {
        if (b == nullptr || tc == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_batch_upload_tc()");
        }
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            sh.ensure_tc();
            rows_h2d(sh, sh.d_tc, tc, static_cast<std::size_t>(sh.n_eq) * (sh.order + 1u), b->n, b->off[i]);
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_get_ptrs(hy_batch *b, hy_batch_ptrs *out)
{
    if (b != nullptr && b->multi) {
        hy::detail::set_last_error("hy_batch_get_ptrs() is not available on a multi-device batch: use the shards");
        return HY_ERR_INVALID_ARG;
    }
    if (b == nullptr || out == nullptr) {
        hy::detail::set_last_error("Null pointer passed to hy_batch_get_ptrs()");
        return HY_ERR_INVALID_ARG;
    }
    const shard &sh = *b->shards[0];
    out->state = sh.d_state;
    out->pars = sh.d_pars;
    out->t_hi = sh.d_t_hi;
    out->t_lo = sh.d_t_lo;
    out->last_h = sh.d_last_h;
    out->tc = sh.d_tc; // null until a step with write_tc / a dense output has been requested
    out->d_out = sh.d_d_out;
    out->step_outcome = reinterpret_cast<int64_t *>(sh.d_step_outcome);
    out->prop_outcome = reinterpret_cast<int64_t *>(sh.d_prop_outcome);
    out->prop_min_h = sh.d_prop_min_h;
    out->prop_max_h = sh.d_prop_max_h;
    out->prop_n_steps = reinterpret_cast<uint64_t *>(sh.d_prop_n_steps);
    return HY_OK;
}

int hy_batch_step(hy_batch *b, const double *max_delta_t, int on_device, int backward, int write_tc)
{
    try {
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        if (on_device && b->multi) {
            throw std::invalid_argument("Device-resident step limits are not available on a multi-device batch");
        }
        if (max_delta_t != nullptr && !on_device) {
            // step(max_delta_ts): NaN limits are rejected (src/taylor_adaptive_batch.cpp:1060-1075).
            for (std::uint32_t i = 0; i < b->n; ++i) {
                if (std::isnan(max_delta_t[i])) {
                    throw std::invalid_argument("Cannot use a nan max_delta_t in the step() function of an adaptive "
                                                "Taylor integrator in batch mode");
                }
            }
        }
        if (b->n_ev != 0u && !b->ev_set) {
            throw std::invalid_argument("hy_batch_set_events() must be called before stepping a batch with event equations");
        }
        std::vector<std::vector<hy_event_rec>> evs(b->shards.size());
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            const double *d_mdt = stage(sh, max_delta_t, on_device, b->off[i], 0);
            if (b->n_ev != 0u) {
                // A batch with event equations: every step detects events (the Taylor coefficients are always written,
                // src/taylor_adaptive_batch.cpp:776); hy_batch_get_events() returns what was found.
                evs[i] = sh.ev_step(d_mdt, backward);
                return;
            }
            dev::run_args R{};
            R.max_delta_t = d_mdt;
            R.default_max_delta_t
                = backward ? -std::numeric_limits<double>::infinity() : std::numeric_limits<double>::infinity();
            R.write_tc = write_tc;
            R.flags = sh.d_flags;
            R.counter = sh.d_counter;
            sh.launch(false, R);
        });
        if (b->n_ev != 0u) {
            // The shards' lists one after the other, with the lanes of the whole batch: lanes ascending.
            b->ev_host.clear();
            for (std::size_t i = 0; i < evs.size(); ++i) {
                for (hy_event_rec r : evs[i]) {
                    r.lane += b->off[i];
                    b->ev_host.push_back(r);
                }
            }
        }
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_propagate_until(hy_batch *b, const double *t_final_hi, const double *t_final_lo, const double *max_delta_t,
                             uint64_t max_steps, int write_tc)
{
    try {
        refuse_events(b);
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        if (t_final_hi == nullptr) {
            throw std::invalid_argument("Null final times passed to hy_batch_propagate_until()");
        }
        check_prop_args(b->n, t_final_hi, t_final_lo, max_delta_t);
        check_prop_times(b, t_final_hi, t_final_lo);
        propagate(b, t_final_hi, t_final_lo, max_delta_t, 0, max_steps, write_tc, nullptr);
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

// propagate_until() on HOST buffers in one call: upload of state / parameters / times, propagation, download of state,
// times, last_h and the per-lane results (the outputs may alias the inputs). On a batch made of shards
// (hy_batch_create_multi(): several devices, or the SAME device listed several times) every shard runs its copies and
// its kernel on its own stream from its own host thread: with k shards on one device the copies of a shard overlap the
// kernels of the others, and only 1 / k of the transfers stays exposed. The checks on the current times are done on the
// caller's arrays (no read-back).
int hy_batch_propagate_until_host(hy_batch *b, const double *state_in, const double *pars, const double *t_hi_in,
                                  const double *t_lo_in, const double *t_final_hi, const double *t_final_lo,
                                  const double *max_delta_t, uint64_t max_steps, double *state, double *t_hi, double *t_lo,
                                  double *last_h, int64_t *outcome, double *min_h, double *max_h, uint64_t *n_steps)
{
    try {
        if (b == nullptr || state_in == nullptr || t_hi_in == nullptr || t_lo_in == nullptr || t_final_hi == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_batch_propagate_until_host()");
        }
        refuse_events(b);
        check_prop_args(b->n, t_final_hi, t_final_lo, max_delta_t);
        check_prop_times_host(b->n, t_hi_in, t_lo_in, t_final_hi, t_final_lo);
        const prop_host io{state_in, pars, t_hi_in, t_lo_in, state, t_hi, t_lo, last_h, outcome, min_h, max_h, n_steps};
        propagate(b, t_final_hi, t_final_lo, max_delta_t, 0, max_steps, 0, &io);
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_propagate_until_dev(hy_batch *b, const double *d_t_final_hi, const double *d_t_final_lo,
                                 const double *d_max_delta_t, uint64_t max_steps, int write_tc, int *any_nf_or_limit)
{
    try {
        refuse_events(b);
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        if (b->multi) {
            throw std::invalid_argument("hy_batch_propagate_until_dev() is not available on a multi-device batch");
        }
        if (d_t_final_hi == nullptr) {
            throw std::invalid_argument("Null final times passed to hy_batch_propagate_until_dev()");
        }
        const dev::run_flags ex = propagate(b, d_t_final_hi, d_t_final_lo, d_max_delta_t, 1, max_steps, write_tc, nullptr);
        if (any_nf_or_limit != nullptr) {
            *any_nf_or_limit = (ex.any_nf != 0u ? 1 : 0) | (ex.any_limit != 0u ? 2 : 0);
        }
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

// propagate_grid() (src/taylor_adaptive_batch.cpp:1545-2055). The reference's algorithm is kept as it is: an
// initial propagate_until(grid[0]) with write_tc, then lock-step iterations of {dense output at every grid point
// covered by the last step; one step clamped to the last grid point}. The per-lane work runs on the device (one
// step launch + three small kernels per iteration); the host only reads the loop flags, and combines those of the
// shards of a sharded batch.
namespace
{

// The argument checks of propagate_grid_impl() (src/taylor_adaptive_batch.cpp:1575-1670); reads the current times back.
void check_grid(hy_batch *b, const double *grid, uint64_t n_pts, const double *max_delta_t)
{
    const std::uint32_t n = b->n;
    if (n_pts == 0u) {
        throw std::invalid_argument("Cannot invoke propagate_grid() in an adaptive Taylor integrator in batch mode "
                                    "if the time grid is empty");
    }
    if (n_pts > 0xffffffffull) {
        throw std::overflow_error("Too many grid points passed to propagate_grid()");
    }
    // The current time must be finite (:1590-1594).
    std::vector<double> t_hi(n), t_lo(n);
    download(b, nullptr, t_hi.data(), t_lo.data(), nullptr);
    for (std::uint32_t i = 0; i < n; ++i) {
        if (!std::isfinite(t_hi[i]) || !std::isfinite(t_lo[i])) {
            throw std::invalid_argument("Cannot invoke propagate_grid() in an adaptive Taylor integrator in "
                                        "batch mode if the current time is not finite");
        }
    }
    if (max_delta_t != nullptr) {
        for (std::uint32_t i = 0; i < n; ++i) {
            if (std::isnan(max_delta_t[i])) {
                throw std::invalid_argument("A nan max_delta_t was passed to the propagate_grid() function of an "
                                            "adaptive Taylor integrator in batch mode");
            }
            if (max_delta_t[i] <= 0) {
                throw std::invalid_argument("A non-positive max_delta_t was passed to the propagate_grid() "
                                            "function of an adaptive Taylor integrator in batch mode");
            }
        }
    }
    // Grid checks, :1619-1656: finite, strictly monotonic, same direction in every lane.
    constexpr auto nf_err_msg
        = "A non-finite time value was passed to propagate_grid() in an adaptive Taylor integrator in batch mode";
    constexpr auto ig_err_msg = "A non-monotonic time grid was passed to propagate_grid() in an adaptive "
                                "Taylor integrator in batch mode";
    const auto batch_nf = [&](std::uint64_t k) {
        return std::any_of(grid + k * n, grid + (k + 1u) * n, [](double t) { return !std::isfinite(t); });
    };
    if (batch_nf(0)) {
        throw std::invalid_argument(nf_err_msg);
    }
    if (n_pts > 1u) {
        // The direction is established from the first two points of lane 0.
        if (batch_nf(1)) {
            throw std::invalid_argument(nf_err_msg);
        }
        if (grid[n] == grid[0]) {
            throw std::invalid_argument(ig_err_msg);
        }
        const bool dir = grid[n] > grid[0];
        for (std::uint64_t k = 1; k < n_pts; ++k) {
            if (k > 1u && batch_nf(k)) {
                throw std::invalid_argument(nf_err_msg);
            }
            for (std::uint32_t i = 0; i < n; ++i) {
                if ((grid[k * n + i] > grid[(k - 1u) * n + i]) != dir) {
                    throw std::invalid_argument(ig_err_msg);
                }
            }
        }
    }
    // The grid must start at the current time (:1660-1670).
    for (std::uint32_t i = 0; i < n; ++i) {
        if (t_hi[i] != grid[i]) {
            throw std::invalid_argument(
                "When invoking propagate_grid(), the first element of the time grid must match the current "
                "time coordinate - however, the first element of the time grid at batch index "
                + std::to_string(i) + " has a value of " + hy::detail::fmt_double(grid[i])
                + ", while the current time coordinate is " + hy::detail::fmt_double(t_hi[i]));
        }
    }
}

// The reference's lock-step loop (src/taylor_adaptive_batch.cpp:1372-1527, :1696-2053) on one shard: the per-lane state
// of dev::lockstep_state and the buffers behind it. An iteration is a step (step(), or an event step), book(), whatever
// the caller launches after the bookkeeping, then read(): one read-back per iteration.
struct lockstep {
    shard &sh;
    dev_ptr<double> lane; // rem_hi, rem_lo, dt_limit, max_delta_t: [4][n]
    dev_ptr<unsigned char> dir;
    dev_ptr<unsigned> d_flags; // [0, 3) those of dev::lockstep_state, [3] one more word for the caller
    dev::lockstep_state L{};
    unsigned flags[4] = {0u, 0u, 0u, 0u}; // as last read back
    const unsigned char *angles = nullptr; // the rows every step reduces (shard::prop_angles()), or null

    // d_tf_hi, d_tf_lo: the target times on the device (d_tf_lo may be null); max_delta_t: host array or null.
    lockstep(shard &s, const double *d_tf_hi, const double *d_tf_lo, const double *max_delta_t)
        : sh(s), lane(dev_alloc<double>(4u * std::size_t(s.n))), dir(dev_alloc<unsigned char>(s.n)),
          d_flags(dev_alloc<unsigned>(4u))
    {
        const std::uint32_t n = sh.n;
        if (max_delta_t != nullptr) {
            HY_CUDA_CHECK(cudaMemcpyAsync(lane.get() + 3u * n, max_delta_t, sizeof(double) * n, cudaMemcpyHostToDevice,
                                          sh.stream));
        }
        L.tf_hi = d_tf_hi;
        L.tf_lo = d_tf_lo;
        L.max_delta_t = max_delta_t != nullptr ? lane.get() + 3u * n : nullptr;
        L.rem_hi = lane.get();
        L.rem_lo = lane.get() + n;
        L.dt_limit = lane.get() + 2u * n;
        L.t_dir = dir.get();
        L.flags = d_flags.get();
    }
    unsigned blocks() const
    {
        return (sh.n + 127u) / 128u;
    }
    // Remaining times, directions, counters and the limit of the first step.
    void init()
    {
        HY_CUDA_CHECK(cudaMemsetAsync(d_flags.get(), 0, sizeof(flags), sh.stream));
        dev::k_lockstep_init<<<blocks(), 128, 0, sh.stream>>>(sh.view(), L, sh.d_prop_min_h, sh.d_prop_max_h,
                                                                sh.d_prop_n_steps);
        HY_CUDA_CHECK(cudaGetLastError());
    }
    // One step of every lane within its dt_limit, with its Taylor coefficients written to sh.d_tc.
    void step()
    {
        dev::run_args R{};
        R.max_delta_t = L.dt_limit;
        R.default_max_delta_t = std::numeric_limits<double>::infinity();
        R.write_tc = 1;
        R.flags = sh.d_flags;
        R.counter = sh.d_counter;
        R.angles = angles;
        sh.launch(false, R);
    }
    // The bookkeeping of the step just taken. All four flag words start it cleared.
    void book()
    {
        HY_CUDA_CHECK(cudaMemsetAsync(d_flags.get(), 0, sizeof(flags), sh.stream));
        dev::k_lockstep_book<<<blocks(), 128, 0, sh.stream>>>(sh.view(), L, sh.d_prop_outcome, sh.d_prop_min_h,
                                                                sh.d_prop_max_h, sh.d_prop_n_steps);
        HY_CUDA_CHECK(cudaGetLastError());
    }
    void read()
    {
        HY_CUDA_CHECK(cudaMemcpyAsync(flags, d_flags.get(), sizeof(flags), cudaMemcpyDeviceToHost, sh.stream));
        HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
    }
    // After an iteration in which a lane went non-finite: the reference returns before the step callback, so the
    // reduction of that step is undone. The reduced rows are evaluated again from the step's Taylor coefficients with
    // the step's h (the same polynomial evaluation as the step kernel's, so the same bits).
    void undo_reduction()
    {
        if (angles == nullptr) {
            return;
        }
        const std::uint32_t n = sh.n;
        dev::k_d_output<<<(n + 127u) / 128u, 128, 0, sh.stream>>>(sh.prog, n, sh.d_tc, sh.d_last_h, sh.d_d_out);
        HY_CUDA_CHECK(cudaGetLastError());
        ++sh.n_launches;
        for (std::uint32_t i = 0; i < sh.n_eq; ++i) {
            if (sh.angles[i] != 0u) {
                HY_CUDA_CHECK(cudaMemcpyAsync(sh.d_state + std::size_t(i) * n, sh.d_d_out + std::size_t(i) * n,
                                              sizeof(double) * n, cudaMemcpyDeviceToDevice, sh.stream));
            }
        }
        HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
    }
};

} // namespace

int hy_batch_check_grid(hy_batch *b, const double *grid, uint64_t n_pts, const double *max_delta_t)
{
    try {
        if (b == nullptr || grid == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_batch_check_grid()");
        }
        check_grid(b, grid, n_pts, max_delta_t);
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

// ------------------------------------------------------------------------------------------------
// Continuous output.
// ------------------------------------------------------------------------------------------------
struct hy_cout {
    int device = 0;
    std::uint32_t n = 0, n_eq = 0, order = 0;
    std::uint64_t n_steps = 0; // recorded iterations; times have n_steps + 2 rows (start, ..., padding)
    dev::program prog{};
    // The Taylor coefficients of the recorded iterations live in slabs of slab_iters iterations each, written in
    // place by the step kernel (no copy, no final re-pack); d_slabs is the device-side table of the slab pointers.
    std::vector<dev_ptr<double>> slabs;
    dev_ptr<double *> d_slabs;
    std::uint32_t slab_iters = 1;
    cudaStream_t stream = nullptr;
    dev_ptr<double> d_t_hi, d_t_lo, d_tm, d_out;
};

// A recording under construction (update_c_out() / make_c_out(), src/taylor_adaptive_batch.cpp:1277-1346): the
// Taylor coefficients of the current iteration go to slot(), commit() appends the times and closes the iteration.
// Plain steps of the device lock-step loop have the step kernel write straight into the slot; append() copies the
// batch's tc array there first, for event steps (on the device, and in the front ends' host lock-step loops through
// hy_cout_rec_append()).
struct hy_cout_rec {
    std::unique_ptr<hy_cout> co;
    dev_ptr<double> d_times; // rows of 2 * n doubles (hi, lo)
    std::size_t times_cap = 0, times_rows = 0, tc_doubles = 0;
    std::uint64_t iter = 0; // committed iterations

    explicit hy_cout_rec(shard &sh);
    double *slot();
    void commit(shard &sh);
    void append(shard &sh);
    hy_cout *finish(shard &sh, const unsigned char *forward);

private:
    void push_times(shard &sh);
};

// Row 0 of the times: the starting times.
hy_cout_rec::hy_cout_rec(shard &sh)
    : co(std::make_unique<hy_cout>()), tc_doubles(static_cast<std::size_t>(sh.n_eq) * (sh.order + 1u) * sh.n)
{
    co->device = sh.device;
    co->n = sh.n;
    co->n_eq = sh.n_eq;
    co->order = sh.order;
    co->prog = sh.prog;
    co->stream = sh.stream;
    // Slabs of about 64 MB (at least one iteration each).
    co->slab_iters = static_cast<std::uint32_t>(
        std::min<std::size_t>(std::max<std::size_t>((std::size_t(64) << 20) / (tc_doubles * sizeof(double)), 1u), 4096u));
    push_times(sh);
}

void hy_cout_rec::push_times(shard &sh)
{
    const std::uint32_t n = sh.n;
    if (times_rows == times_cap) {
        const std::size_t new_cap = std::max<std::size_t>(2u * times_cap, 64u);
        auto nt = dev_alloc<double>(2u * n * new_cap);
        if (d_times != nullptr) {
            HY_CUDA_CHECK(cudaMemcpyAsync(nt.get(), d_times.get(), sizeof(double) * 2u * n * times_rows,
                                          cudaMemcpyDeviceToDevice, sh.stream));
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        }
        d_times = std::move(nt);
        times_cap = new_cap;
    }
    double *blk = d_times.get() + 2u * n * times_rows;
    HY_CUDA_CHECK(cudaMemcpyAsync(blk, sh.d_t_hi, sizeof(double) * n, cudaMemcpyDeviceToDevice, sh.stream));
    HY_CUDA_CHECK(cudaMemcpyAsync(blk + n, sh.d_t_lo, sizeof(double) * n, cudaMemcpyDeviceToDevice, sh.stream));
    ++times_rows;
}

// The Taylor coefficients of the current iteration; a slab is allocated when the iteration starts one.
double *hy_cout_rec::slot()
{
    if (iter / co->slab_iters == co->slabs.size()) {
        co->slabs.push_back(dev_alloc<double>(tc_doubles * co->slab_iters));
    }
    return co->slabs[iter / co->slab_iters].get() + (iter % co->slab_iters) * tc_doubles;
}

void hy_cout_rec::commit(shard &sh)
{
    push_times(sh);
    ++iter;
}

// (The rows of the state variables come first in the batch's tc array; those of event equations are not recorded.)
void hy_cout_rec::append(shard &sh)
{
    HY_CUDA_CHECK(cudaMemcpyAsync(slot(), sh.d_tc, sizeof(double) * tc_doubles, cudaMemcpyDeviceToDevice, sh.stream));
    commit(sh);
}

// make_c_out() (:1277-1317): forward[lane] != 0 for lanes integrated forwards in time (the padding row of the times is
// +-inf by direction). Null if nothing was recorded.
hy_cout *hy_cout_rec::finish(shard &sh, const unsigned char *forward)
{
    if (iter == 0u) {
        return nullptr;
    }
    const std::uint32_t n = sh.n;
    co->n_steps = iter;
    const std::size_t rows = iter + 2u;
    co->d_t_hi = dev_alloc<double>(rows * n);
    co->d_t_lo = dev_alloc<double>(rows * n);
    co->d_tm = dev_alloc<double>(n);
    co->d_out = dev_alloc<double>(static_cast<std::size_t>(sh.n_eq) * n);
    HY_CUDA_CHECK(cudaMemcpy2DAsync(co->d_t_hi.get(), sizeof(double) * n, d_times.get(), sizeof(double) * 2u * n,
                                    sizeof(double) * n, iter + 1u, cudaMemcpyDeviceToDevice, sh.stream));
    HY_CUDA_CHECK(cudaMemcpy2DAsync(co->d_t_lo.get(), sizeof(double) * n, d_times.get() + n, sizeof(double) * 2u * n,
                                    sizeof(double) * n, iter + 1u, cudaMemcpyDeviceToDevice, sh.stream));
    std::vector<double *> slabs(co->slabs.size());
    std::transform(co->slabs.begin(), co->slabs.end(), slabs.begin(), [](const dev_ptr<double> &p) { return p.get(); });
    co->d_slabs = dev_alloc<double *>(slabs.size());
    HY_CUDA_CHECK(cudaMemcpyAsync(co->d_slabs.get(), slabs.data(), sizeof(double *) * slabs.size(), cudaMemcpyHostToDevice,
                                  sh.stream));
    HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
    std::vector<double> pad(n), zero(n, 0.);
    for (std::uint32_t i = 0; i < n; ++i) {
        pad[i] = forward[i] != 0 ? std::numeric_limits<double>::infinity() : -std::numeric_limits<double>::infinity();
    }
    HY_CUDA_CHECK(cudaMemcpy(co->d_t_hi.get() + (rows - 1u) * n, pad.data(), sizeof(double) * n, cudaMemcpyHostToDevice));
    HY_CUDA_CHECK(cudaMemcpy(co->d_t_lo.get() + (rows - 1u) * n, zero.data(), sizeof(double) * n, cudaMemcpyHostToDevice));
    return co.release();
}

int hy_cout_rec_begin(hy_batch *b, hy_cout_rec **out)
{
    try {
        if (b == nullptr || out == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_cout_rec_begin()");
        }
        if (b->multi) {
            throw hy::detail::not_implemented_error("Continuous output is not available on a multi-device batch");
        }
        *out = nullptr;
        shard &sh = *b->shards[0];
        device_guard guard(sh.device);
        auto r = std::make_unique<hy_cout_rec>(sh);
        HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        *out = r.release();
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_cout_rec_append(hy_batch *b, hy_cout_rec *r)
{
    try {
        if (b == nullptr || b->multi || r == nullptr || r->co == nullptr || r->co->n != b->n
            || b->shards[0]->d_tc == nullptr) {
            throw std::invalid_argument("Invalid arguments passed to hy_cout_rec_append() (the last step must have "
                                        "written its Taylor coefficients)");
        }
        shard &sh = *b->shards[0];
        device_guard guard(sh.device);
        r->append(sh);
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

void hy_cout_rec_destroy(hy_cout_rec *r)
{
    delete r;
}

// The recorder is destroyed either way.
int hy_cout_rec_finish(hy_batch *b, hy_cout_rec *rp, const unsigned char *forward, hy_cout **out)
{
    std::unique_ptr<hy_cout_rec> r(rp);
    try {
        if (b == nullptr || rp == nullptr || forward == nullptr || out == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_cout_rec_finish()");
        }
        *out = nullptr;
        shard &sh = *b->shards[0];
        device_guard guard(sh.device);
        *out = r->finish(sh, forward);
        HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

// ------------------------------------------------------------------------------------------------
// The lock-step propagations: propagate_until() with continuous output (hy_batch_propagate_until_cout{,_cb}()),
// propagate_grid() (hy_batch_propagate_grid()), and both for a batch with event equations
// (hy_batch_propagate_until_ev(), hy_batch_propagate_grid_ev()). One driver runs the reference's lock-step loop
// (src/taylor_adaptive_batch.cpp:1372-1527, :1696-2053) over the shards of a batch, with the bookkeeping on the device.
// A batch with events takes event steps: the host takes part in an iteration only when some lane produced an event
// record, receives the records with their absolute times and hands back the terminal-event decisions.
// ------------------------------------------------------------------------------------------------
namespace
{

struct callback_abort {
};

// The lock-step loop over every shard of a batch. The reference's loop runs over the whole batch, so the shards run in
// lock-step and the loop's exits are decided from the flags of all of them. cb == null: plain steps (lockstep::step());
// otherwise event steps, with cb the events' callback.
struct lockstep_run {
    struct part {
        std::unique_ptr<lockstep> ls;
        dev_ptr<double> d_tf;           // target times of propagate_until() (hi, lo)
        std::vector<hy_event_rec> recs; // live records of the iteration, lanes local to the shard
        std::vector<double> t;          // their absolute times: [2][recs.size()] (hi, lo)
        std::vector<std::uint32_t> go;  // local lanes whose terminal-event callback continues
        dev_ptr<unsigned char> d_buf;   // staging of records, times and lanes
        std::size_t buf_bytes = 0;

        unsigned char *buf(std::size_t bytes)
        {
            if (bytes > buf_bytes) {
                buf_bytes = std::max(bytes, 2u * buf_bytes);
                d_buf = dev_alloc<unsigned char>(buf_bytes);
            }
            return d_buf.get();
        }
    };
    hy_batch *b;
    hy_event_callback cb;
    void *user;
    std::vector<part> sh; // one per shard of b
    std::vector<hy_event_rec> recs;
    std::vector<double> t_hi, t_lo;
    std::vector<unsigned char> cont;
    std::uint64_t iter = 0; // iterations taken
    bool started = false;   // some iteration's bookkeeping ran in this call
    unsigned done = 0;      // lanes at their target in the last iteration
    bool nf = false;        // a lane went non-finite in the last iteration
    bool stop = false;      // a terminal event without a callback, or whose callback returned false, fired

    lockstep_run(hy_batch *b_, hy_event_callback cb_, void *user_) : b(b_), cb(cb_), user(user_), sh(b_->shards.size()) {}

    // The lock-step states towards per-lane final times (host arrays; t_final_lo and max_delta_t may be null), with
    // each shard's reduced rows.
    void until(const double *t_final_hi, const double *t_final_lo, const double *max_delta_t)
    {
        for_each_shard(b, [&](shard &s, std::size_t i) {
            const std::size_t off = b->off[i];
            part &e = sh[i];
            e.d_tf = dev_alloc<double>(2u * std::size_t(s.n));
            HY_CUDA_CHECK(cudaMemcpyAsync(e.d_tf.get(), t_final_hi + off, sizeof(double) * s.n, cudaMemcpyHostToDevice,
                                          s.stream));
            if (t_final_lo != nullptr) {
                HY_CUDA_CHECK(cudaMemcpyAsync(e.d_tf.get() + s.n, t_final_lo + off, sizeof(double) * s.n,
                                              cudaMemcpyHostToDevice, s.stream));
            }
            e.ls = std::make_unique<lockstep>(s, e.d_tf.get(), t_final_lo != nullptr ? e.d_tf.get() + s.n : nullptr,
                                              max_delta_t != nullptr ? max_delta_t + off : nullptr);
            e.ls->angles = s.prop_angles();
            e.ls->init();
            e.ls->read();
        });
        check_overflow("propagate_until()");
    }
    // After init() and read(): the remaining time of every lane must be representable. fn names the caller.
    void check_overflow(const char *fn) const
    {
        for (const auto &e : sh) {
            if (e.ls->flags[2] != 0u) {
                throw std::invalid_argument(std::string("The final time passed to the ") + fn
                                            + " function of an adaptive Taylor integrator in batch mode results in an "
                                              "overflow condition");
            }
        }
    }

    // The event step of every shard, then the callbacks (if there are records) and the terminal-event decisions.
    void event_step()
    {
        for_each_shard(b, [&](shard &s, std::size_t i) {
            part &e = sh[i];
            e.recs = s.ev_step(e.ls->L.dt_limit, 0);
            const auto k = static_cast<std::uint32_t>(e.recs.size());
            e.t.resize(2u * std::size_t(k));
            if (k != 0u) {
                unsigned char *buf = e.buf(k * (sizeof(hy_event_rec) + 2u * sizeof(double)));
                auto *d_recs = reinterpret_cast<hy_event_rec *>(buf);
                auto *d_t = reinterpret_cast<double *>(buf + std::size_t(k) * sizeof(hy_event_rec));
                HY_CUDA_CHECK(cudaMemcpyAsync(d_recs, e.recs.data(), sizeof(hy_event_rec) * k, cudaMemcpyHostToDevice,
                                              s.stream));
                dev::k_ev_times<<<(k + 127u) / 128u, 128, 0, s.stream>>>(s.view(), d_recs, k, d_t, d_t + k);
                HY_CUDA_CHECK(cudaGetLastError());
                ++s.n_launches;
                HY_CUDA_CHECK(cudaMemcpyAsync(e.t.data(), d_t, sizeof(double) * 2u * k, cudaMemcpyDeviceToHost, s.stream));
                HY_CUDA_CHECK(cudaStreamSynchronize(s.stream));
            }
        });
        // The shards' records one after the other, with the lanes of the whole batch (as hy_batch_step() lists them).
        recs.clear();
        t_hi.clear();
        t_lo.clear();
        for (std::size_t i = 0; i < sh.size(); ++i) {
            const std::size_t k = sh[i].recs.size();
            for (std::size_t j = 0; j < k; ++j) {
                hy_event_rec r = sh[i].recs[j];
                r.lane += b->off[i];
                recs.push_back(r);
                t_hi.push_back(sh[i].t[j]);
                t_lo.push_back(sh[i].t[k + j]);
            }
        }
        if (recs.empty()) {
            return;
        }
        cont.assign(recs.size(), 0u);
        const int r = cb(user, recs.data(), t_hi.data(), t_lo.data(), static_cast<std::uint32_t>(recs.size()),
                         cont.data());
        std::size_t k = 0;
        for (auto &e : sh) {
            e.go.clear();
            for (const auto &rec : e.recs) {
                if (rec.terminal != 0) {
                    if (cont[k] != 0u) {
                        e.go.push_back(rec.lane);
                    } else {
                        stop = true;
                    }
                }
                ++k;
            }
        }
        // The decisions are applied whatever the callback returned, like the front ends' loops do lane by lane.
        for_each_shard(b, [&](shard &s, std::size_t i) {
            part &e = sh[i];
            const auto n_go = static_cast<std::uint32_t>(e.go.size());
            if (n_go != 0u) {
                auto *d_lanes = reinterpret_cast<std::uint32_t *>(e.buf(sizeof(std::uint32_t) * n_go));
                HY_CUDA_CHECK(cudaMemcpyAsync(d_lanes, e.go.data(), sizeof(std::uint32_t) * n_go,
                                              cudaMemcpyHostToDevice, s.stream));
                dev::k_ev_continue<<<(n_go + 127u) / 128u, 128, 0, s.stream>>>(s.view(), d_lanes, n_go);
                HY_CUDA_CHECK(cudaGetLastError());
                ++s.n_launches;
            }
            if (r < 0 && !started) {
                // Aborted before any bookkeeping: the per-lane results read as before the first step.
                dev::k_fill_outcome<<<(s.n + 255u) / 256u, 256, 0, s.stream>>>(s.d_prop_outcome, s.n, 0);
                dev::k_fill_double<<<(s.n + 255u) / 256u, 256, 0, s.stream>>>(s.d_prop_min_h, s.n, 0.);
                HY_CUDA_CHECK(cudaGetLastError());
            }
            HY_CUDA_CHECK(cudaStreamSynchronize(s.stream));
        });
        if (r < 0) {
            throw callback_abort{};
        }
    }

    // One iteration of every shard: the step, the bookkeeping, then after_book(shard, i) if given and the flags read
    // back.
    void iterate(const std::function<void(shard &, std::size_t)> &after_book = nullptr)
    {
        if (cb != nullptr) {
            event_step();
        }
        for_each_shard(b, [&](shard &s, std::size_t i) {
            lockstep &ls = *sh[i].ls;
            if (cb == nullptr) {
                ls.step();
            }
            ls.book();
            if (after_book) {
                after_book(s, i);
            }
            ls.read();
        });
        started = true;
        done = 0u;
        nf = false;
        for (const auto &e : sh) {
            done += e.ls->flags[0];
            nf = nf || e.ls->flags[1] != 0u;
        }
        ++iter;
    }

    void undo_reduction()
    {
        for_each_shard(b, [&](shard &, std::size_t i) { sh[i].ls->undo_reduction(); });
    }

    void fill_outcome(long long oc)
    {
        for_each_shard(b, [&](shard &s, std::size_t) {
            dev::k_fill_outcome<<<(s.n + 255u) / 256u, 256, 0, s.stream>>>(s.d_prop_outcome, s.n, oc);
            HY_CUDA_CHECK(cudaGetLastError());
            HY_CUDA_CHECK(cudaStreamSynchronize(s.stream));
        });
    }

    // propagate_until() from the lock-step states already initialised: iterations up to the loop's exits, in the
    // reference's order. Every iteration that ends with finite states is recorded by rec (shard 0's recorder) if given,
    // and followed by the step callback step_cb(step_user) if given.
    void run_until(std::uint64_t max_steps, hy_cout_rec *rec, hy_step_callback step_cb, void *step_user)
    {
        shard &s0 = *b->shards[0];
        // Plain steps record in place: the step kernel writes the coefficients of every iteration straight into their
        // slot of the recording (a copy would move the whole tc array once per iteration), and the batch's own tc array
        // is put back however the loop ends. The tc array of an event step also holds the event rows: it is copied.
        // (The recorder allocates its slabs and times on shard 0's device.)
        const bool in_place = rec != nullptr && cb == nullptr;
        if (in_place) {
            device_guard guard(s0.device);
            s0.ensure_tc();
        }
        struct tc_restore {
            shard &sh;
            double *const own; // null: nothing to put back
            ~tc_restore()
            {
                if (own != nullptr) {
                    sh.d_tc = own;
                }
            }
        } tc{s0, in_place ? s0.d_tc : nullptr};
        while (true) {
            if (in_place) {
                device_guard guard(s0.device);
                s0.d_tc = rec->slot();
            }
            iterate();
            if (nf) {
                undo_reduction();
                break; // non-finite state: this iteration is not recorded (:1462-1467)
            }
            if (rec != nullptr) {
                // update_c_out(), :1320-1346
                device_guard guard(s0.device);
                if (in_place) {
                    rec->commit(s0);
                } else {
                    rec->append(s0);
                }
            }
            if (step_cb != nullptr) {
                // The step callback (:1476-1500), before the exit tests like in the reference.
                HY_CUDA_CHECK(cudaStreamSynchronize(s0.stream));
                const int r = step_cb(step_user);
                if (r < 0) {
                    throw callback_abort{};
                }
                if (r == 0) {
                    fill_outcome(HY_OUTCOME_CB_STOP);
                    break;
                }
            }
            if (stop || done == b->n) {
                break; // a stopping terminal event, or every lane reached its final time
            }
            if (iter == max_steps) {
                fill_outcome(HY_OUTCOME_STEP_LIMIT);
                break;
            }
        }
        if (in_place) {
            // The batch's own tc array ends up with the coefficients of the last step taken, like m_tc in the reference.
            device_guard guard(s0.device);
            HY_CUDA_CHECK(cudaMemcpyAsync(tc.own, s0.d_tc, sizeof(double) * rec->tc_doubles, cudaMemcpyDeviceToDevice,
                                          s0.stream));
        }
    }
};

// propagate_grid() on every shard of a batch: per shard its columns of the grid, its block of the output and its
// cursors, and the driver L with the lock-step states towards the last grid point. Every shard takes every iteration
// while some lane of some shard has grid points left (a shard whose lanes are all at their target takes zero-length
// steps, as those lanes do inside one device), and an iteration in which a lane of any shard goes non-finite is
// sampled by no shard.
struct grid_run {
    struct part {
        dev_ptr<double> d_grid, d_out; // [n_pts][n], [n_pts][n_eq][n]
        dev_ptr<std::uint32_t> d_idx;
    };
    hy_batch *b;
    std::uint64_t n_pts;
    const double *max_delta_t;
    std::vector<part> p; // one per shard of b
    lockstep_run L;

    // Stages the grid by column and fills every shard's output with NaN.
    grid_run(hy_batch *b_, const double *grid, std::uint64_t n_pts_, const double *max_delta_t_, hy_event_callback cb,
             void *user)
        : b(b_), n_pts(n_pts_), max_delta_t(max_delta_t_), p(b_->shards.size()), L(b_, cb, user)
    {
        for_each_shard(b, [&](shard &s, std::size_t i) {
            const std::size_t n_out = static_cast<std::size_t>(n_pts) * s.n_eq * s.n;
            p[i].d_grid = dev_alloc<double>(n_pts * s.n);
            p[i].d_out = dev_alloc<double>(n_out);
            p[i].d_idx = dev_alloc<std::uint32_t>(s.n);
            rows_h2d(s, p[i].d_grid.get(), grid, n_pts, b->n, b->off[i]);
            dev::k_fill_double<<<static_cast<unsigned>((n_out + 255u) / 256u), 256, 0, s.stream>>>(
                p[i].d_out.get(), n_out, std::numeric_limits<double>::quiet_NaN());
            HY_CUDA_CHECK(cudaGetLastError());
            HY_CUDA_CHECK(cudaStreamSynchronize(s.stream));
        });
    }
    const double *mdt(std::size_t i) const
    {
        return max_delta_t != nullptr ? max_delta_t + b->off[i] : nullptr;
    }
    // Up to the first grid point (:1697-1706: propagate_until(grid[0])).
    void first_leg(const double *grid, std::uint64_t max_steps)
    {
        if (L.cb == nullptr) {
            // A zero-length step when the time is already there: it brings the Taylor coefficients up to date. The
            // reference calls no step callback there: no reduction.
            propagate(b, grid, nullptr, max_delta_t, 0, max_steps, 1, nullptr, false);
            return;
        }
        // With the events and their callbacks.
        for_each_shard(b, [&](shard &s, std::size_t i) {
            L.sh[i].ls = std::make_unique<lockstep>(s, p[i].d_grid.get(), nullptr, mdt(i));
            L.sh[i].ls->init();
        });
        L.run_until(max_steps, nullptr, nullptr, nullptr);
    }
    // After the propagation to grid[0]: whether every lane of every shard reached it. If not, the counters are reset
    // and the outcomes kept (:1709-1722).
    bool first_leg_done()
    {
        std::vector<long long> oc(b->n);
        for_each_shard(b, [&](shard &s, std::size_t i) {
            rows_d2h(s, oc.data(), s.d_prop_outcome, 1u, b->n, b->off[i]);
            HY_CUDA_CHECK(cudaStreamSynchronize(s.stream));
        });
        if (std::all_of(oc.begin(), oc.end(), [](long long v) { return v == HY_OUTCOME_TIME_LIMIT; })) {
            return true;
        }
        for_each_shard(b, [&](shard &s, std::size_t) {
            const unsigned gb = (s.n + 127u) / 128u;
            dev::k_fill_double<<<gb, 128, 0, s.stream>>>(s.d_prop_min_h, s.n, std::numeric_limits<double>::infinity());
            dev::k_fill_double<<<gb, 128, 0, s.stream>>>(s.d_prop_max_h, s.n, 0.);
            HY_CUDA_CHECK(cudaGetLastError());
            HY_CUDA_CHECK(cudaMemsetAsync(s.d_prop_n_steps, 0, sizeof(unsigned long long) * s.n, s.stream));
            HY_CUDA_CHECK(cudaStreamSynchronize(s.stream));
        });
        return false;
    }
    // Grid point 0 is the current state, every cursor starts at 1; the lock-step states towards the last grid point
    // (each shard's reduced rows: angles[i]), and the grid points the zero-length interval before the first step covers.
    void start(const std::vector<const unsigned char *> &angles)
    {
        for_each_shard(b, [&](shard &s, std::size_t i) {
            part &q = p[i];
            HY_CUDA_CHECK(cudaMemcpyAsync(q.d_out.get(), s.d_state, sizeof(double) * s.n_eq * s.n,
                                          cudaMemcpyDeviceToDevice, s.stream));
            const std::vector<std::uint32_t> first(s.n, 1u);
            HY_CUDA_CHECK(cudaMemcpyAsync(q.d_idx.get(), first.data(), sizeof(std::uint32_t) * s.n,
                                          cudaMemcpyHostToDevice, s.stream));
            L.sh[i].ls = std::make_unique<lockstep>(s, q.d_grid.get() + (n_pts - 1u) * s.n, nullptr, mdt(i));
            L.sh[i].ls->angles = angles[i];
            L.sh[i].ls->init();
            sample(s, i);
            L.sh[i].ls->read();
        });
        L.check_overflow("propagate_grid()");
    }
    // Dense output at the grid points the shard's last step covered, and the cursors past them. The word the lock-step
    // state leaves to its caller is set when some lane has grid points left.
    void sample(shard &s, std::size_t i)
    {
        const part &q = p[i];
        const lockstep &ls = *L.sh[i].ls;
        const dev::grid_state G{q.d_grid.get(), static_cast<std::uint32_t>(n_pts), q.d_out.get(), q.d_idx.get(),
                                ls.d_flags.get() + 3};
        const unsigned gb = ls.blocks();
        dev::k_grid_sample<<<dim3(gb, s.n_eq), 128, 0, s.stream>>>(s.prog, s.view(), G, ls.L);
        dev::k_grid_advance<<<gb, 128, 0, s.stream>>>(s.view(), G, ls.L);
        HY_CUDA_CHECK(cudaGetLastError());
    }
    bool any_flag(unsigned w) const
    {
        return std::any_of(L.sh.begin(), L.sh.end(), [w](const lockstep_run::part &e) { return e.ls->flags[w] != 0u; });
    }
    // The lock-step loop (:1770-2053). One shard samples right after its bookkeeping, where the kernels' own check of
    // the non-finite flag is batch-wide: one read-back per iteration. More shards combine their non-finite flags on the
    // host first, then sample and read the flags again.
    void loop(std::uint64_t max_steps)
    {
        const bool one = p.size() == 1u;
        L.stop = false;
        std::uint64_t iter = 0;
        while (any_flag(3)) {
            L.iterate([&](shard &s, std::size_t i) {
                if (one) {
                    sample(s, i);
                }
            });
            if (L.nf) {
                // Non-finite state: nothing further is written, and the reduction of this step is undone (:1973-1978).
                L.undo_reduction();
                return;
            }
            if (!one) {
                for_each_shard(b, [&](shard &s, std::size_t i) {
                    sample(s, i);
                    L.sh[i].ls->read();
                });
            }
            if (++iter == max_steps) {
                L.fill_outcome(HY_OUTCOME_STEP_LIMIT);
                return;
            }
            if (L.stop) {
                return; // a stopping terminal event, once the grid points of this step are written
            }
        }
    }
    // Every shard's block of the output into the caller's [n_pts][n_eq][batch] array.
    int finish(double *out)
    {
        for_each_shard(b, [&](shard &s, std::size_t i) {
            rows_d2h(s, out, p[i].d_out.get(), static_cast<std::size_t>(n_pts) * s.n_eq, b->n, b->off[i]);
            HY_CUDA_CHECK(cudaStreamSynchronize(s.stream));
        });
        return HY_OK;
    }
};

// The checks every event propagation makes on its batch and callback.
void check_ev_batch(const hy_batch *b, hy_event_callback cb, const char *fn)
{
    if (b == nullptr || cb == nullptr) {
        throw std::invalid_argument(std::string("Null pointer passed to ") + fn);
    }
    if (b->n_ev == 0u) {
        throw std::invalid_argument(std::string(fn) + " needs a batch with event equations");
    }
    if (!b->ev_set) {
        throw std::invalid_argument("hy_batch_set_events() must be called before stepping a batch with event equations");
    }
    for (const auto &s : b->shards) {
        if (s->angles_on) {
            throw hy::detail::not_implemented_error("The angle reducer does not run inside the propagation of a batch "
                                                    "with event equations");
        }
    }
}

// propagate_until() of every lane of a checked batch: event steps with the events' callback cb, or plain steps with the
// step callback step_cb (either may be null; user goes to the one given), recorded into *c_out if c_out is not null.
int propagate_until_lockstep(hy_batch *b, const double *t_final_hi, const double *t_final_lo,
                             const double *max_delta_t, uint64_t max_steps, hy_event_callback cb,
                             hy_step_callback step_cb, void *user, hy_cout **c_out)
{
    try {
        lockstep_run L(b, cb, user);
        L.until(t_final_hi, t_final_lo, max_delta_t);
        shard &s0 = *b->shards[0];
        std::unique_ptr<hy_cout_rec> rec;
        if (c_out != nullptr) {
            device_guard guard(s0.device);
            rec = std::make_unique<hy_cout_rec>(s0);
        }
        L.run_until(max_steps, rec.get(), step_cb, user);
        if (rec != nullptr) {
            device_guard guard(s0.device);
            std::vector<unsigned char> forward(s0.n);
            HY_CUDA_CHECK(cudaMemcpyAsync(forward.data(), L.sh[0].ls->L.t_dir, s0.n, cudaMemcpyDeviceToHost, s0.stream));
            HY_CUDA_CHECK(cudaStreamSynchronize(s0.stream));
            *c_out = rec->finish(s0, forward.data());
            HY_CUDA_CHECK(cudaStreamSynchronize(s0.stream));
        }
        return HY_OK;
    } catch (const callback_abort &) {
        hy::detail::set_last_error("A host callback aborted the propagation");
        return HY_ERR_CALLBACK;
    }
}

// propagate_grid() of every lane of a checked batch: event steps with the events' callback cb, or plain steps with the
// angle reducer.
int propagate_grid_lockstep(hy_batch *b, const double *grid, uint64_t n_pts, const double *max_delta_t,
                            uint64_t max_steps, hy_event_callback cb, void *user, double *out)
{
    try {
        // (Before any grid work: a refused angle list leaves the batch untouched. Event batches have none.)
        std::vector<const unsigned char *> angles(b->shards.size());
        for (std::size_t i = 0; i < b->shards.size(); ++i) {
            angles[i] = b->shards[i]->prop_angles();
        }
        grid_run G(b, grid, n_pts, max_delta_t, cb, user);
        G.first_leg(grid, max_steps);
        if (!G.first_leg_done()) {
            return G.finish(out);
        }
        G.start(angles);
        G.loop(max_steps);
        return G.finish(out);
    } catch (const callback_abort &) {
        hy::detail::set_last_error("A host callback aborted the propagation");
        return HY_ERR_CALLBACK;
    }
}

} // namespace

int hy_batch_propagate_until_cout(hy_batch *b, const double *t_final_hi, const double *t_final_lo,
                                  const double *max_delta_t, uint64_t max_steps, hy_cout **out)
{
    return hy_batch_propagate_until_cout_cb(b, t_final_hi, t_final_lo, max_delta_t, max_steps, nullptr, nullptr, out);
}

int hy_batch_propagate_until_cout_cb(hy_batch *b, const double *t_final_hi, const double *t_final_lo,
                                     const double *max_delta_t, uint64_t max_steps, hy_step_callback cb, void *user,
                                     hy_cout **out)
{
    try {
        refuse_events(b);
        if (b != nullptr && b->multi) {
            throw hy::detail::not_implemented_error("Continuous output is not available on a multi-device batch");
        }
        if (b == nullptr || t_final_hi == nullptr || out == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_batch_propagate_until_cout()");
        }
        *out = nullptr;
        // (The step callback runs with the batch's device current.)
        device_guard guard(b->shards[0]->device);
        check_prop_args(b->n, t_final_hi, t_final_lo, max_delta_t);
        return propagate_until_lockstep(b, t_final_hi, t_final_lo, max_delta_t, max_steps, nullptr, cb, user, out);
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_propagate_until_ev(hy_batch *b, const double *t_final_hi, const double *t_final_lo,
                                const double *max_delta_t, uint64_t max_steps, hy_event_callback cb, void *user,
                                hy_cout **c_out)
{
    try {
        check_ev_batch(b, cb, "hy_batch_propagate_until_ev()");
        if (t_final_hi == nullptr) {
            throw std::invalid_argument("Null final times passed to hy_batch_propagate_until_ev()");
        }
        if (c_out != nullptr) {
            *c_out = nullptr;
            if (b->multi) {
                throw hy::detail::not_implemented_error("Continuous output is not available on a multi-device batch");
            }
        }
        check_prop_args(b->n, t_final_hi, t_final_lo, max_delta_t);
        check_prop_times(b, t_final_hi, t_final_lo);
        return propagate_until_lockstep(b, t_final_hi, t_final_lo, max_delta_t, max_steps, cb, nullptr, user, c_out);
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_propagate_grid(hy_batch *b, const double *grid, uint64_t n_pts, const double *max_delta_t,
                            uint64_t max_steps, double *out)
{
    try {
        refuse_events(b);
        if (b == nullptr || grid == nullptr || out == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_batch_propagate_grid()");
        }
        check_grid(b, grid, n_pts, max_delta_t);
        return propagate_grid_lockstep(b, grid, n_pts, max_delta_t, max_steps, nullptr, nullptr, out);
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_propagate_grid_ev(hy_batch *b, const double *grid, uint64_t n_pts, const double *max_delta_t,
                               uint64_t max_steps, hy_event_callback cb, void *user, double *out)
{
    try {
        check_ev_batch(b, cb, "hy_batch_propagate_grid_ev()");
        if (grid == nullptr || out == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_batch_propagate_grid_ev()");
        }
        check_grid(b, grid, n_pts, max_delta_t);
        return propagate_grid_lockstep(b, grid, n_pts, max_delta_t, max_steps, cb, user, out);
    } catch (...) {
        return translate_exception();
    }
}

int hy_cout_eval(hy_cout *c, const double *tm, double *out)
{
    try {
        if (c == nullptr || tm == nullptr || out == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_cout_eval()");
        }
        for (std::uint32_t i = 0; i < c->n; ++i) {
            if (!std::isfinite(tm[i])) {
                throw std::invalid_argument("Cannot compute the continuous output in batch mode for the batch index "
                                            + std::to_string(i) + " at the non-finite time "
                                            + hy::detail::fmt_double(tm[i]));
            }
        }
        device_guard guard(c->device);
        HY_CUDA_CHECK(cudaMemcpyAsync(c->d_tm.get(), tm, sizeof(double) * c->n, cudaMemcpyHostToDevice, c->stream));
        dev::k_cout_eval<<<(c->n + 127u) / 128u, 128, 0, c->stream>>>(
            c->prog, c->n, static_cast<std::uint32_t>(c->n_steps + 2u), c->d_slabs.get(), c->slab_iters,
            c->d_t_hi.get(), c->d_t_lo.get(), c->d_tm.get(), c->d_out.get());
        HY_CUDA_CHECK(cudaGetLastError());
        HY_CUDA_CHECK(cudaMemcpyAsync(out, c->d_out.get(), sizeof(double) * static_cast<std::size_t>(c->n_eq) * c->n,
                                      cudaMemcpyDeviceToHost, c->stream));
        HY_CUDA_CHECK(cudaStreamSynchronize(c->stream));
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_cout_get_bounds(const hy_cout *c, double *lb, double *ub)
{
    try {
        if (c == nullptr || lb == nullptr || ub == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_cout_get_bounds()");
        }
        device_guard guard(c->device);
        HY_CUDA_CHECK(cudaMemcpy(lb, c->d_t_hi.get(), sizeof(double) * c->n, cudaMemcpyDeviceToHost));
        HY_CUDA_CHECK(cudaMemcpy(ub, c->d_t_hi.get() + c->n_steps * c->n, sizeof(double) * c->n, cudaMemcpyDeviceToHost));
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_cout_download(const hy_cout *c, double *times_hi, double *times_lo, double *tcs)
{
    try {
        if (c == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_cout_download()");
        }
        device_guard guard(c->device);
        const std::size_t n = c->n, rows = static_cast<std::size_t>(c->n_steps) + 2u;
        if (times_hi != nullptr) {
            HY_CUDA_CHECK(cudaMemcpy(times_hi, c->d_t_hi.get(), sizeof(double) * rows * n, cudaMemcpyDeviceToHost));
        }
        if (times_lo != nullptr) {
            HY_CUDA_CHECK(cudaMemcpy(times_lo, c->d_t_lo.get(), sizeof(double) * rows * n, cudaMemcpyDeviceToHost));
        }
        if (tcs != nullptr) {
            // One iteration = [n_eq][order + 1][batch] doubles; the slabs hold slab_iters iterations each, the last
            // one possibly fewer.
            const std::size_t it_doubles = static_cast<std::size_t>(c->n_eq) * (c->order + 1u) * n;
            for (std::size_t s = 0; s < c->slabs.size(); ++s) {
                const std::size_t first = s * c->slab_iters;
                if (first >= c->n_steps) {
                    break;
                }
                const std::size_t count = std::min<std::size_t>(c->slab_iters, c->n_steps - first);
                HY_CUDA_CHECK(cudaMemcpy(tcs + first * it_doubles, c->slabs[s].get(), sizeof(double) * count * it_doubles,
                                         cudaMemcpyDeviceToHost));
            }
        }
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

uint64_t hy_cout_n_steps(const hy_cout *c)
{
    return c != nullptr ? c->n_steps : 0u;
}

void hy_cout_destroy(hy_cout *c)
{
    delete c;
}

int hy_batch_d_output(hy_batch *b, const double *tau, double *out)
{
    try {
        if (b == nullptr || tau == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_batch_d_output()");
        }
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            const double *d_tau = stage(sh, tau, 0, b->off[i], 0);
            sh.ensure_tc();
            dev::k_d_output<<<(sh.n + 127u) / 128u, 128, 0, sh.stream>>>(sh.prog, sh.n, sh.d_tc, d_tau, sh.d_d_out);
            HY_CUDA_CHECK(cudaGetLastError());
            ++sh.n_launches;
            rows_d2h(sh, out, sh.d_d_out, sh.n_eq, b->n, b->off[i]);
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

namespace
{

// k_taylor_map on one shard, device-resident dx / out.
void taylor_map_launch(shard &sh, std::uint32_t n_orig, std::uint32_t m, const double *d_dx, double *d_out)
{
    const std::uint32_t chunk = std::min(m, dev::TMAP_CHUNK);
    dev::k_taylor_map<<<(sh.n + dev::TMAP_THREADS - 1u) / dev::TMAP_THREADS, dev::TMAP_THREADS,
                        sizeof(double) * chunk * dev::TMAP_THREADS, sh.stream>>>(sh.d_state, sh.n, n_orig, m, d_dx,
                                                                                 d_out);
    HY_CUDA_CHECK(cudaGetLastError());
    ++sh.n_launches;
}

// Host form: dx staged into d_tmap[0, m * n), the result read back from d_tmap[m * n, (m + n_orig) * n).
void taylor_map_host(shard &sh, std::uint32_t n_orig, std::uint32_t m, const double *dx, double *out,
                     std::size_t pitch, std::size_t off)
{
    const std::size_t need = static_cast<std::size_t>(m + n_orig) * sh.n;
    if (sh.tmap_doubles < need) {
        if (sh.d_tmap != nullptr) {
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
            HY_CUDA_CHECK(cudaFree(sh.d_tmap));
            sh.d_tmap = nullptr;
            sh.tmap_doubles = 0;
        }
        sh.d_tmap = sh.dalloc<double>(need);
        sh.tmap_doubles = need;
    }
    double *d_dx = sh.d_tmap, *d_out = sh.d_tmap + static_cast<std::size_t>(m) * sh.n;
    rows_h2d(sh, d_dx, dx, m, pitch, off);
    taylor_map_launch(sh, n_orig, m, d_dx, d_out);
    rows_d2h(sh, out, d_out, n_orig, pitch, off);
    HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
}

} // namespace

int hy_batch_eval_taylor_map(hy_batch *b, uint32_t n_orig_sv, uint32_t n_args, const double *dx, double *out,
                             int on_device)
{
    try {
        if (b == nullptr || dx == nullptr || out == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_batch_eval_taylor_map()");
        }
        if (n_orig_sv == 0u || n_args == 0u
            || static_cast<std::uint64_t>(n_orig_sv) * (1u + static_cast<std::uint64_t>(n_args)) != b->n_eq) {
            throw std::invalid_argument(
                "Invalid sizes passed to hy_batch_eval_taylor_map(): " + std::to_string(n_orig_sv)
                + " original state variables and " + std::to_string(n_args)
                + " arguments do not make a variational system of order 1 with " + std::to_string(b->n_eq)
                + " equations");
        }
        if (on_device && b->multi) {
            throw std::invalid_argument(
                "Device-resident arrays are not available for the Taylor map of a multi-device batch");
        }
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            if (on_device) {
                // (Asynchronous on the batch's stream, like the other device-resident entry points.)
                taylor_map_launch(sh, n_orig_sv, n_args, dx, out);
            } else {
                taylor_map_host(sh, n_orig_sv, n_args, dx, out, b->n, b->off[i]);
            }
        });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

/* ---- E. events ---- */
int hy_batch_set_events(hy_batch *b, uint32_t n_te, const int32_t *dirs, const double *cooldowns, double tol)
{
    try {
        if (b == nullptr || dirs == nullptr || (n_te != 0u && cooldowns == nullptr)) {
            throw std::invalid_argument("Null pointer passed to hy_batch_set_events()");
        }
        if (b->n_ev == 0u) {
            throw std::invalid_argument("This batch was built from a program without event equations");
        }
        if (n_te > b->n_ev) {
            throw std::invalid_argument("The number of terminal events exceeds the number of event equations");
        }
        for (std::uint32_t k = 0; k < b->n_ev; ++k) {
            if (dirs[k] < -1 || dirs[k] > 1) {
                throw std::invalid_argument("Invalid value selected for the direction of an event");
            }
        }
        for (std::uint32_t k = 0; k < n_te; ++k) {
            if (!std::isfinite(cooldowns[k])) {
                throw std::invalid_argument("Cannot set a non-finite cooldown value for a terminal event");
            }
        }
        // (Directions, cooldowns and tolerance are per event, not per lane: every shard gets them all.)
        for_each_shard(b, [&](shard &sh, std::size_t) {
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
            sh.ev_setup(n_te, dirs, cooldowns, tol);
        });
        b->n_te = n_te;
        b->ev_set = true;
        b->ev_host.clear();
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

uint32_t hy_batch_n_events(const hy_batch *b)
{
    return b == nullptr ? 0u : static_cast<uint32_t>(b->ev_host.size());
}

int hy_batch_get_events(const hy_batch *b, hy_event_rec *out, uint32_t cap)
{
    if (b == nullptr || (out == nullptr && cap != 0u)) {
        hy::detail::set_last_error("Null pointer passed to hy_batch_get_events()");
        return HY_ERR_INVALID_ARG;
    }
    const std::size_t m = std::min<std::size_t>(cap, b->ev_host.size());
    std::copy(b->ev_host.begin(), b->ev_host.begin() + static_cast<std::ptrdiff_t>(m), out);
    return HY_OK;
}

int hy_batch_download_tc_events(hy_batch *b, double *out)
{
    try {
        if (b == nullptr || out == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_batch_download_tc_events()");
        }
        if (b->n_ev == 0u
            || std::any_of(b->shards.begin(), b->shards.end(), [](const auto &sh) { return sh->d_tc == nullptr; })) {
            throw std::invalid_argument("No Taylor coefficients of event equations are available");
        }
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            // (The rows of the event equations follow those of the state variables.)
            const std::size_t rows = static_cast<std::size_t>(sh.order + 1u) * sh.n_ev;
            rows_d2h(sh, out, sh.d_tc + static_cast<std::size_t>(sh.order + 1u) * sh.n * sh.n_eq, rows, b->n, b->off[i]);
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_reset_cooldowns(hy_batch *b, int64_t lane)
{
    try {
        if (b == nullptr) {
            throw std::invalid_argument("Null batch");
        }
        if (!b->ev_set) {
            throw std::invalid_argument("No events are defined for this integrator");
        }
        if (lane >= static_cast<int64_t>(b->n)) {
            throw std::invalid_argument("Cannot reset the cooldowns at batch index " + std::to_string(lane)
                                        + ": the batch size for this integrator is only " + std::to_string(b->n));
        }
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            const auto lo = static_cast<int64_t>(b->off[i]);
            const std::size_t m = static_cast<std::size_t>(b->n_te) * sh.n;
            if (m == 0u || (lane >= 0 && (lane < lo || lane >= lo + sh.n))) {
                return;
            }
            dev::k_ev_reset_cd<<<static_cast<unsigned>((m + 255u) / 256u), 256, 0, sh.stream>>>(
                sh.eva, sh.n, lane < 0 ? 0xffffffffu : static_cast<std::uint32_t>(lane - lo));
            HY_CUDA_CHECK(cudaGetLastError());
        });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

// The cooldown state [n_te][batch] is gathered / scattered by columns: every shard keeps its lanes' active flags as
// [n_te][lanes] and the time spent and the cooldown as [n_te][2][lanes].
int hy_batch_get_cooldowns(hy_batch *b, uint8_t *active, double *spent, double *cooldown)
{
    try {
        if (b == nullptr || !b->ev_set) {
            throw std::invalid_argument("No events are defined for this integrator");
        }
        if (b->n_te != 0u && (active == nullptr || spent == nullptr || cooldown == nullptr)) {
            throw std::invalid_argument("Null pointer passed to hy_batch_get_cooldowns()");
        }
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            rows_d2h(sh, active, sh.eva.cd_on, b->n_te, b->n, b->off[i]);
            for (std::uint32_t k = 0; k < b->n_te; ++k) {
                const std::size_t row = static_cast<std::size_t>(k) * b->n;
                rows_d2h(sh, spent + row, sh.eva.cd + static_cast<std::size_t>(2u * k) * sh.n, 1u, b->n, b->off[i]);
                rows_d2h(sh, cooldown + row, sh.eva.cd + static_cast<std::size_t>(2u * k + 1u) * sh.n, 1u, b->n, b->off[i]);
            }
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_set_cooldowns(hy_batch *b, const uint8_t *active, const double *spent, const double *cooldown)
{
    try {
        if (b == nullptr || !b->ev_set) {
            throw std::invalid_argument("No events are defined for this integrator");
        }
        if (b->n_te != 0u && (active == nullptr || spent == nullptr || cooldown == nullptr)) {
            throw std::invalid_argument("Null pointer passed to hy_batch_set_cooldowns()");
        }
        for_each_shard(b, [&](shard &sh, std::size_t i) {
            rows_h2d(sh, sh.eva.cd_on, active, b->n_te, b->n, b->off[i]);
            for (std::uint32_t k = 0; k < b->n_te; ++k) {
                const std::size_t row = static_cast<std::size_t>(k) * b->n;
                rows_h2d(sh, sh.eva.cd + static_cast<std::size_t>(2u * k) * sh.n, spent + row, 1u, b->n, b->off[i]);
                rows_h2d(sh, sh.eva.cd + static_cast<std::size_t>(2u * k + 1u) * sh.n, cooldown + row, 1u, b->n, b->off[i]);
            }
            HY_CUDA_CHECK(cudaStreamSynchronize(sh.stream));
        });
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_batch_launch_count(const hy_batch *b, uint64_t *n_launches)
{
    if (b == nullptr || n_launches == nullptr) {
        hy::detail::set_last_error("Null pointer passed to hy_batch_launch_count()");
        return HY_ERR_INVALID_ARG;
    }
    *n_launches = 0u;
    for (const auto &sh : b->shards) {
        *n_launches += sh->n_launches;
    }
    return HY_OK;
}

} // extern "C"
