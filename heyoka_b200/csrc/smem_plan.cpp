// See smem_plan.hpp.
#include "smem_plan.hpp"

#include <algorithm>
#include <cstring>
#include <map>
#include <numeric>
#include <stdexcept>
#include <utility>

namespace heyoka_b200::detail
{

namespace
{

// How one op uses u variables at order n: `now` = read at order n only, `hist` = read at lower orders too.
struct op_uses {
    std::vector<std::uint32_t> now, hist;
    bool self_hist = false;
};

op_uses uses_of(const hy_program &p, const hy_op &op)
{
    op_uses u;
    const auto nary = [&](bool hist) {
        for (std::uint32_t k = 0; k < op.b; ++k) {
            const auto ref = p.args[op.a + k];
            if (HY_REF_KIND(ref) == HY_REF_VAR) {
                (hist ? u.hist : u.now).push_back(HY_REF_IDX(ref));
            }
        }
    };
    switch (op.opcode) {
        case HY_OP_SUM:
            nary(false);
            break;
        case HY_OP_SUM_SQ:
            nary(true);
            break;
        case HY_OP_SUB_VV:
            u.now = {op.a, op.b};
            break;
        case HY_OP_SUB_VN:
        case HY_OP_SUB_VP:
        case HY_OP_DIV_VN:
        case HY_OP_DIV_VP:
        case HY_OP_NEG:
            u.now = {op.a};
            break;
        case HY_OP_SUB_NV:
        case HY_OP_SUB_PV:
        case HY_OP_MUL_NV:
        case HY_OP_MUL_PV:
            u.now = {op.b};
            break;
        case HY_OP_MUL_VV:
            u.hist = {op.a, op.b};
            break;
        case HY_OP_DIV_VV:
            u.now = {op.a};
            u.hist = {op.b};
            u.self_hist = true;
            break;
        case HY_OP_DIV_NV:
        case HY_OP_DIV_PV:
            u.hist = {op.b};
            u.self_hist = true;
            break;
        case HY_OP_SQUARE:
            u.hist = {op.a};
            break;
        case HY_OP_SQRT:
            u.now = {op.a};
            u.self_hist = true;
            break;
        case HY_OP_POW_VN:
        case HY_OP_POW_VP:
        case HY_OP_EXP:
        case HY_OP_LOG:
            u.hist = {op.a};
            u.self_hist = true;
            break;
        case HY_OP_SIN:
        case HY_OP_COS:
        case HY_OP_TANH:
            // op.c is the hidden dependency: read at lower orders only, but it needs its history.
            u.hist = {op.a};
            break;
        case HY_OP_SIGMOID:
            u.hist = {op.a};
            u.self_hist = true;
            break;
        case HY_OP_RELU:
            // Reads the order-0 coefficient of its argument at every order: the argument keeps its history.
            u.hist = {op.a};
            break;
        case HY_OP_RELUP:
            u.now = {op.a};
            break;
        default:
            break;
    }
    return u;
}

// One schedulable work item: an elementary op, or a fused group of them.
struct item {
    hy_op op;                        // for fused items: op.opcode = HY_FOP_*, op.a = offset into aux
    std::uint32_t dst_u = 0;         // u variable defined (elementary ops)
    std::vector<std::uint32_t> defs; // u variables this item defines
    std::vector<std::uint32_t> deps; // u variables read at the current order, defined by OTHER items
    std::uint32_t level = 0;
    std::uint32_t first_op = 0;      // position of the first member op in the program (stable ordering)
    std::uint32_t svo = 0;           // offset into svout (0 = none)
};

} // namespace

smem_plan make_smem_plan(const hy_program &p, bool fuse, bool fuse_sv, bool spill_private)
{
    smem_plan pl;
    const auto n_eq = p.n_eq, n_uvars = p.n_uvars, order = p.order;
    const auto n_ops = n_uvars - n_eq;

    // ---- history analysis ----
    std::vector<char> hist(n_uvars, 0);
    std::vector<std::vector<std::uint32_t>> users(n_uvars); // ops (indices) reading each u variable explicitly
    for (std::uint32_t i = 0; i < n_ops; ++i) {
        const auto &op = p.ops[i];
        const auto u = uses_of(p, op);
        for (const auto v : u.hist) {
            hist[v] = 1;
            users[v].push_back(i);
        }
        for (const auto v : u.now) {
            users[v].push_back(i);
        }
        if (u.self_hist) {
            hist[n_eq + i] = 1;
        }
        if (op.opcode == HY_OP_SIN || op.opcode == HY_OP_COS || op.opcode == HY_OP_TANH
            || op.opcode == HY_OP_SIGMOID) {
            hist[op.c] = 1;
            users[op.c].push_back(i); // keeps hidden dependencies out of any fusion
        }
    }
    std::vector<char> is_sv_def(n_uvars, 0);
    for (const auto ref : p.sv_defs) {
        if (HY_REF_KIND(ref) == HY_REF_VAR) {
            is_sv_def[HY_REF_IDX(ref)] = 1;
        }
    }

    // ---- superinstructions: the gravitational pair interaction of model::nbody ----
    // Pattern (src/model/nbody.cpp:97-153 after decomposition):
    //   d_k = sub(x_k^j, x_k^i), k = 0..2;  r2 = sum_sq(d_0, d_1, d_2);  q = pow(r2, alpha);
    //   f = c1 * q | -q | q;  m_k = d_k * f (either operand order);  optionally n_k = c2_k * m_k.
    // All of it depends, at the current order, only on state variables, so one thread can run the whole chain
    // for a pair. Every u variable keeps its own row and its own recurrence (bit-identical results).
    std::vector<char> fused(n_ops, 0);
    std::vector<char> dropped(n_uvars, 0); // u variables that are never stored (recomputed inside a superinstruction)
    std::vector<char> in_global(n_uvars, 0); // rows private to a superinstruction that live in the overflow tape
    std::vector<item> items;
    // aux entries that hold u-variable indices, to be translated into row references once slots are assigned
    std::vector<std::size_t> aux_is_u;
    struct fused_out {
        std::size_t aux_pos;
        std::uint32_t u[6];
    };
    std::vector<fused_out> fused_outs;
    const auto op_of = [&](std::uint32_t u) -> const hy_op & { return p.ops[u - n_eq]; };
    const auto only_users = [&](std::uint32_t u, std::vector<std::uint32_t> allowed) {
        std::sort(allowed.begin(), allowed.end());
        for (const auto x : users[u]) {
            if (!std::binary_search(allowed.begin(), allowed.end(), x)) {
                return false;
            }
        }
        return true;
    };
    std::vector<std::pair<double, std::uint32_t>> pow_tabs; // (alpha, index of its table in the constant pool)
    if (fuse) {
        for (std::uint32_t qi = 0; qi < n_ops; ++qi) {
            const auto &qop = p.ops[qi];
            if (qop.opcode != HY_OP_POW_VN || qop.a < n_eq) {
                continue;
            }
            const auto r2u = qop.a;
            const auto &sop = op_of(r2u);
            if (sop.opcode != HY_OP_SUM_SQ || sop.b != 3u || fused[r2u - n_eq]) {
                continue;
            }
            std::uint32_t du[3];
            bool ok = true;
            for (std::uint32_t k = 0; k < 3u && ok; ++k) {
                const auto ref = p.args[sop.a + k];
                ok = HY_REF_KIND(ref) == HY_REF_VAR && HY_REF_IDX(ref) >= n_eq;
                if (ok) {
                    du[k] = HY_REF_IDX(ref);
                    const auto &dop = op_of(du[k]);
                    ok = dop.opcode == HY_OP_SUB_VV && dop.a < n_eq && dop.b < n_eq && !fused[du[k] - n_eq];
                }
            }
            if (!ok || du[0] == du[1] || du[1] == du[2] || du[0] == du[2]) {
                continue;
            }
            const auto qu = n_eq + qi;
            // r2 is only read by the pow.
            if (!only_users(r2u, {qi}) || is_sv_def[r2u]) {
                continue;
            }
            // f: the single user of q that scales it, or q itself.
            std::uint32_t fu = qu, fkind = 0 /* 0: q itself, 1: c1 * q, 2: -q */, c1 = 0;
            if (users[qu].size() == 1u) {
                const auto &fop = p.ops[users[qu][0]];
                if (fop.opcode == HY_OP_MUL_NV && fop.b == qu) {
                    fu = n_eq + users[qu][0];
                    fkind = 1;
                    c1 = fop.a;
                } else if (fop.opcode == HY_OP_NEG && fop.a == qu) {
                    fu = n_eq + users[qu][0];
                    fkind = 2;
                }
            }
            if (is_sv_def[qu] || is_sv_def[fu]) {
                continue;
            }
            // m_k: the three products d_k * f. The users of f must be exactly these products, and every d_k
            // must only be read by the sum_sq and by its product.
            std::uint32_t mu[3] = {0, 0, 0};
            std::vector<std::uint32_t> f_users;
            for (std::uint32_t k = 0; k < 3u && ok; ++k) {
                std::uint32_t found = 0, cnt = 0;
                for (const auto x : users[du[k]]) {
                    const auto &mop = p.ops[x];
                    if (mop.opcode == HY_OP_MUL_VV
                        && ((mop.a == du[k] && mop.b == fu) || (mop.b == du[k] && mop.a == fu))) {
                        found = x;
                        ++cnt;
                    }
                }
                ok = cnt == 1u && only_users(du[k], {r2u - n_eq, found}) && !is_sv_def[du[k]] && !fused[found];
                mu[k] = n_eq + found;
                f_users.push_back(found);
            }
            if (!ok || !only_users(fu, f_users) || (fu != qu && !only_users(qu, {fu - n_eq}))) {
                continue;
            }
            // All three products must have the same operand order (d * f or f * d): the pairing of the
            // convolution indices depends on it.
            {
                const bool o0 = op_of(mu[0]).a == du[0], o1 = op_of(mu[1]).a == du[1], o2 = op_of(mu[2]).a == du[2];
                if (o0 != o1 || o1 != o2) {
                    continue;
                }
            }
            // Optional second scaling n_k = c2_k * m_k: fused when every m_k has exactly one such reader
            // (m_k keeps its own row: other readers, e.g. the sums, come at later levels).
            std::uint32_t nu[3] = {0, 0, 0}, c2[3] = {0, 0, 0};
            bool have_n = true;
            for (std::uint32_t k = 0; k < 3u; ++k) {
                std::uint32_t cnt = 0;
                for (const auto x : users[mu[k]]) {
                    const auto &nop = p.ops[x];
                    if (nop.opcode == HY_OP_MUL_NV && nop.b == mu[k] && !fused[x]) {
                        nu[k] = n_eq + x;
                        c2[k] = nop.a;
                        ++cnt;
                    }
                }
                have_n = have_n && cnt == 1u;
            }

            // The device code writes m_k / n_k as single-slot rows: they must not be history rows.
            for (std::uint32_t k = 0; k < 3u; ++k) {
                ok = ok && !hist[mu[k]] && (!have_n || !hist[nu[k]]);
            }
            if (!ok) {
                continue;
            }

            // Build the fused item.
            item it;
            it.op.opcode = HY_FOP_NBODY_PAIR;
            it.op.a = static_cast<std::uint32_t>(pl.aux.size());
            it.op.b = fkind;
            it.op.c = have_n ? 1u : 0u;
            it.first_op = du[0] - n_eq;
            const auto push_u = [&](std::uint32_t u) {
                aux_is_u.push_back(pl.aux.size());
                pl.aux.push_back(u);
            };
            for (std::uint32_t k = 0; k < 3u; ++k) {
                const auto &dop = op_of(du[k]);
                push_u(dop.a);
                push_u(dop.b);
                push_u(du[k]);
            }
            push_u(r2u);
            push_u(qu);
            pl.aux.push_back(qop.b); // exponent (constant index)
            pl.aux.push_back(qop.c); // order-0 evaluation algorithm
            // (f is never stored: f^[j] = c1 q^[j] / -q^[j] is recomputed on the fly.) Index in the constant pool
            // of the table j * (alpha + 1) of the pow recurrence (shared by the pairs with the same exponent).
            {
                const double alpha = p.consts[qop.b];
                std::uint32_t tab_idx = 0;
                bool found = false;
                for (const auto &[a_bits, idx] : pow_tabs) {
                    if (std::memcmp(&a_bits, &alpha, sizeof(double)) == 0) {
                        tab_idx = idx;
                        found = true;
                    }
                }
                if (!found) {
                    tab_idx = static_cast<std::uint32_t>(p.consts.size() + pl.extra_consts.size());
                    const double ap1 = alpha + 1.;
                    for (std::uint32_t j = 0; j <= order; ++j) {
                        pl.extra_consts.push_back(static_cast<double>(j) * ap1);
                    }
                    pow_tabs.emplace_back(alpha, tab_idx);
                }
                pl.aux.push_back(tab_idx);
            }
            pl.aux.push_back(c1);
            for (std::uint32_t k = 0; k < 3u; ++k) {
                const auto &mop = op_of(mu[k]);
                push_u(mu[k]);
                pl.aux.push_back(mop.a == du[k] ? 0u : 1u); // operand order of the product (d * f or f * d)
                if (have_n) {
                    push_u(nu[k]);
                } else {
                    pl.aux.push_back(0u);
                }
                pl.aux.push_back(have_n ? c2[k] : 0u);
            }
            // svout offsets of m_0..2, n_0..2 (filled in after level scheduling).
            fused_outs.push_back({pl.aux.size(), {mu[0], mu[1], mu[2], have_n ? nu[0] : 0u, have_n ? nu[1] : 0u,
                                                  have_n ? nu[2] : 0u}});
            pl.aux.insert(pl.aux.end(), 6u, 0u);
            if (fu != qu) {
                dropped[fu] = 1;
            }
            if (spill_private) {
                in_global[r2u] = 1;
                in_global[qu] = 1;
            }
            std::vector<std::uint32_t> members{du[0], du[1], du[2], r2u, qu, mu[0], mu[1], mu[2]};
            if (fu != qu) {
                members.push_back(fu);
            }
            if (have_n) {
                members.insert(members.end(), {nu[0], nu[1], nu[2]});
            }
            for (const auto m : members) {
                fused[m - n_eq] = 1;
                it.defs.push_back(m);
            }
            items.push_back(std::move(it));
            ++pl.n_fused;
        }
    }

    // ---- the remaining elementary ops ----
    for (std::uint32_t i = 0; i < n_ops; ++i) {
        if (fused[i]) {
            continue;
        }
        item it;
        it.op = p.ops[i];
        it.dst_u = n_eq + i;
        it.defs = {n_eq + i};
        it.first_op = i;
        const auto u = uses_of(p, p.ops[i]);
        for (const auto v : u.now) {
            if (v >= n_eq) {
                it.deps.push_back(v);
            }
        }
        for (const auto v : u.hist) {
            // convolution operands are read at order n too (e.g. b^[n] c^[0])
            if (v >= n_eq) {
                it.deps.push_back(v);
            }
        }
        items.push_back(std::move(it));
    }

    // ---- slot assignment ----
    // Odd history stride: consecutive history rows then start in different shared-memory bank groups.
    const std::uint32_t hstride = (order + 1u) | 1u;
    std::vector<std::uint32_t> row(n_uvars, 0);
    std::uint32_t next = 0, gnext = 0;
    const auto alloc = [&](std::uint32_t kind, std::uint32_t n) {
        const auto r = (kind << ROW_SLOT_BITS) | next;
        next += n;
        return r;
    };
    const auto assign = [&](std::uint32_t i) {
        if (dropped[i]) {
            row[i] = 0u;
        } else if (in_global[i]) {
            // Slot index in the overflow tape (only the superinstruction that owns the row knows about it).
            row[i] = (ROW_H << ROW_SLOT_BITS) | gnext;
            gnext += hstride;
        } else if (hist[i]) {
            row[i] = alloc(ROW_H, hstride);
        } else if (i < n_eq) {
            row[i] = alloc(ROW_SV, 2u);
        } else {
            row[i] = alloc(ROW_T, 1u);
        }
    };
    // The threads of a warp run consecutive items of a level, and at any instant they all touch the row that
    // plays the same role in their own item: rows are laid out so that those rows are hstride (odd) or 1 slots
    // apart, i.e. in different bank groups for 8 consecutive threads (a slot is 16 bytes with 2 lanes per warp).
    //   state variables: one pad slot per group of 6 (x, y, z, vx, vy, vz of one particle), so that the same
    //                    coordinate of different particles is an odd number of slots apart;
    //   superinstructions: role-major (all the dx rows, then all the dy rows, ...), in execution order;
    //   elementary ops: program order (= execution order inside a level for ops of the same kind).
    for (std::uint32_t i = 0; i < n_eq; ++i) {
        assign(i);
        if (n_eq % 6u == 0u && i % 6u == 5u) {
            next += 1u;
        }
    }
    std::sort(items.begin(), items.end(), [](const item &x, const item &y) { return x.first_op < y.first_op; });
    {
        std::vector<std::uint8_t> done(items.size(), 0);
        for (std::size_t k = 0; k < items.size(); ++k) {
            if (done[k] || items[k].op.opcode < HY_FOP_FIRST) {
                continue;
            }
            std::vector<std::size_t> grp;
            for (std::size_t k2 = k; k2 < items.size(); ++k2) {
                if (!done[k2] && items[k2].op.opcode == items[k].op.opcode
                    && items[k2].defs.size() == items[k].defs.size()) {
                    grp.push_back(k2);
                    done[k2] = 1;
                }
            }
            for (std::size_t r = 0; r < items[k].defs.size(); ++r) {
                for (const auto g : grp) {
                    assign(items[g].defs[r]);
                }
            }
        }
        for (std::size_t k = 0; k < items.size(); ++k) {
            if (!done[k]) {
                for (const auto d : items[k].defs) {
                    assign(d);
                }
            }
        }
    }
    if (next >= (1u << ROW_SLOT_BITS)) {
        throw std::overflow_error("The Taylor tape is too large");
    }
    pl.n_slots = next;
    pl.n_gslots = gnext;
    pl.sv_rows.assign(row.begin(), row.begin() + n_eq);

    // ---- n-ary argument table and state-variable definitions with row references ----
    pl.args = p.args;
    for (auto &ref : pl.args) {
        if (HY_REF_KIND(ref) == HY_REF_VAR) {
            ref = HY_REF(HY_REF_VAR, row[HY_REF_IDX(ref)]);
        }
    }
    pl.sv_defs = p.sv_defs;
    for (auto &ref : pl.sv_defs) {
        if (HY_REF_KIND(ref) == HY_REF_VAR) {
            ref = HY_REF(HY_REF_VAR, row[HY_REF_IDX(ref)]);
        }
    }

    for (const auto pos : aux_is_u) {
        pl.aux[pos] = row[pl.aux[pos]];
    }

    // ---- level scheduling: an item runs one level after the last producer of what it reads at the current
    // order. (The reference's taylor_segment_dc(), src/taylor_02.cpp:105-207, cuts the BFS-sorted list
    // greedily; levels give the same or fewer synchronisation points. Hidden dependencies are not dependencies.)
    std::vector<std::uint32_t> producer(n_uvars, ~0u);
    for (std::uint32_t k = 0; k < items.size(); ++k) {
        for (const auto d : items[k].defs) {
            producer[d] = k;
        }
    }
    std::sort(items.begin(), items.end(), [](const item &x, const item &y) { return x.first_op < y.first_op; });
    for (std::uint32_t k = 0; k < items.size(); ++k) {
        for (const auto d : items[k].defs) {
            producer[d] = k;
        }
    }
    // Items sorted by first_op: producers of elementary ops come earlier in program order, fused items only
    // depend on state variables. One forward pass is enough, but iterate to a fixed point to be safe.
    for (bool changed = true; changed;) {
        changed = false;
        for (auto &it : items) {
            std::uint32_t lvl = 0;
            for (const auto d : it.deps) {
                lvl = std::max(lvl, items[producer[d]].level + 1u);
            }
            if (lvl != it.level) {
                it.level = lvl;
                changed = true;
            }
        }
    }
    std::uint32_t n_levels = 0;
    for (const auto &it : items) {
        n_levels = std::max(n_levels, it.level + 1u);
    }
    pl.n_segments = n_levels;

    // ---- state-variable propagation fused into the producers (see smem_plan.hpp) ----
    {
        // Highest level at which each state variable is read at the current order.
        std::vector<std::int64_t> sv_read_level(n_eq, -1);
        for (const auto &it : items) {
            std::vector<std::uint32_t> reads;
            if (it.op.opcode >= HY_FOP_FIRST) {
                for (const auto d : it.defs) {
                    const auto u = uses_of(p, op_of(d));
                    reads.insert(reads.end(), u.now.begin(), u.now.end());
                    reads.insert(reads.end(), u.hist.begin(), u.hist.end());
                }
            } else {
                const auto u = uses_of(p, it.op);
                reads.insert(reads.end(), u.now.begin(), u.now.end());
                reads.insert(reads.end(), u.hist.begin(), u.hist.end());
            }
            for (const auto v : reads) {
                if (v < n_eq) {
                    sv_read_level[v] = std::max<std::int64_t>(sv_read_level[v], it.level);
                }
            }
        }
        pl.sv_cover.assign(n_eq, 0u);
        pl.sv_parent.assign(n_eq, 0u);
        std::vector<std::vector<std::uint32_t>> direct(n_uvars);   // u -> state variables with rhs u
        std::vector<std::vector<std::uint32_t>> children(n_eq);    // s -> depth-2 state variables with rhs s
        for (std::uint32_t s2 = 0; s2 < n_eq; ++s2) {
            const auto ref = p.sv_defs[s2];
            if (fuse_sv && HY_REF_KIND(ref) == HY_REF_VAR && HY_REF_IDX(ref) >= n_eq && !dropped[HY_REF_IDX(ref)]) {
                direct[HY_REF_IDX(ref)].push_back(s2);
                pl.sv_cover[s2] = 1u;
            }
        }
        for (std::uint32_t s2 = 0; s2 < n_eq; ++s2) {
            const auto ref = p.sv_defs[s2];
            if (HY_REF_KIND(ref) != HY_REF_VAR || HY_REF_IDX(ref) >= n_eq) {
                continue;
            }
            const auto s1 = HY_REF_IDX(ref);
            if (pl.sv_cover[s1] != 1u) {
                continue;
            }
            // x_s2^[n+2] is written while order n is being processed, into the slot that holds x_s2^[n] unless
            // s2 keeps its whole history: nobody may still read x_s2^[n] at or after the producer's level.
            const auto prod_level = items[producer[HY_REF_IDX(p.sv_defs[s1])]].level;
            if (!hist[s2] && sv_read_level[s2] >= static_cast<std::int64_t>(prod_level)) {
                continue;
            }
            children[s1].push_back(s2);
            pl.sv_cover[s2] = 2u;
            pl.sv_parent[s2] = s1;
        }
        for (std::uint32_t s2 = 0; s2 < n_eq; ++s2) {
            if (pl.sv_cover[s2] == 0u) {
                pl.sv_phase.push_back(s2);
            }
        }
        // svout lists.
        std::vector<std::uint32_t> svo_of_u(n_uvars, 0u);
        pl.svout.push_back(0u); // offset 0 is "none"
        for (std::uint32_t u = n_eq; u < n_uvars; ++u) {
            if (direct[u].empty()) {
                continue;
            }
            svo_of_u[u] = static_cast<std::uint32_t>(pl.svout.size());
            const auto cnt_pos = pl.svout.size();
            pl.svout.push_back(0u);
            std::uint32_t cnt = 0;
            for (const auto s1 : direct[u]) {
                pl.svout.insert(pl.svout.end(), {s1, row[s1], 1u});
                ++cnt;
                for (const auto s2 : children[s1]) {
                    pl.svout.insert(pl.svout.end(), {s2, row[s2], 2u});
                    ++cnt;
                }
            }
            pl.svout[cnt_pos] = cnt;
        }
        for (const auto &fo : fused_outs) {
            for (std::uint32_t k = 0; k < 6u; ++k) {
                pl.aux[fo.aux_pos + k] = fo.u[k] != 0u ? svo_of_u[fo.u[k]] : 0u;
            }
        }
        for (auto &it : items) {
            it.svo = it.op.opcode >= HY_FOP_FIRST ? 0u : svo_of_u[it.dst_u];
        }
    }

    // A sum whose terms are all single-slot rows: the argument table entries are the slots themselves.
    for (auto &it : items) {
        if (it.op.opcode != HY_OP_SUM) {
            continue;
        }
        bool all_t = true;
        for (std::uint32_t k = 0; k < it.op.b; ++k) {
            const auto ref = p.args[it.op.a + k];
            all_t = all_t && HY_REF_KIND(ref) == HY_REF_VAR && HY_REF_IDX(ref) >= n_eq && !hist[HY_REF_IDX(ref)];
        }
        if (all_t) {
            it.op.opcode = HY_FOP_SUM_T;
        }
    }

    // ---- emit: level by level, grouped by opcode inside a level (warp-uniform control flow) ----
    pl.seg_offsets.push_back(0);
    for (std::uint32_t lvl = 0; lvl < n_levels; ++lvl) {
        std::vector<const item *> cur;
        for (const auto &it : items) {
            if (it.level == lvl) {
                cur.push_back(&it);
            }
        }
        std::stable_sort(cur.begin(), cur.end(),
                         [](const item *x, const item *y) { return x->op.opcode < y->op.opcode; });
        pl.max_seg_width = std::max<std::uint32_t>(pl.max_seg_width, static_cast<std::uint32_t>(cur.size()));
        for (const auto *it : cur) {
            auto op = it->op;
            const auto var = [&](std::uint32_t &f) { f = row[f]; };
            switch (op.opcode) {
                case HY_OP_SUB_VV:
                case HY_OP_MUL_VV:
                case HY_OP_DIV_VV:
                    var(op.a);
                    var(op.b);
                    break;
                case HY_OP_SUB_VN:
                case HY_OP_SUB_VP:
                case HY_OP_DIV_VN:
                case HY_OP_DIV_VP:
                case HY_OP_NEG:
                case HY_OP_SQUARE:
                case HY_OP_SQRT:
                case HY_OP_POW_VN:
                case HY_OP_POW_VP:
                case HY_OP_EXP:
                case HY_OP_LOG:
                    var(op.a);
                    break;
                case HY_OP_SUB_NV:
                case HY_OP_SUB_PV:
                case HY_OP_MUL_NV:
                case HY_OP_MUL_PV:
                case HY_OP_DIV_NV:
                case HY_OP_DIV_PV:
                    var(op.b);
                    break;
                case HY_OP_SIN:
                case HY_OP_COS:
                case HY_OP_TANH:
                case HY_OP_SIGMOID:
                    var(op.a);
                    var(op.c);
                    break;
                case HY_OP_RELU:
                case HY_OP_RELUP:
                    var(op.a);
                    break;
                default:
                    // SUM / SUM_SQ / CFUNC go through the argument table, TIME has no operands, fused
                    // items carry row references in aux.
                    break;
            }
            pl.ops.push_back(op);
            pl.dst.push_back(op.opcode == HY_FOP_NBODY_PAIR ? 0u : row[it->dst_u]);
            pl.svo.push_back(it->svo);
        }
        pl.seg_offsets.push_back(static_cast<std::uint32_t>(pl.ops.size()));
    }

    return pl;
}

} // namespace heyoka_b200::detail
