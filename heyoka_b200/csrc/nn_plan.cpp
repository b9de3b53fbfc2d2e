// See nn_plan.hpp.
#include "nn_plan.hpp"

#include <algorithm>
#include <map>

namespace heyoka_b200::detail
{

namespace
{

struct fail {
    std::string why;
};

// b + sum_k c_k * base_k, base_k = a state variable or the output of an activation.
struct linear_form {
    double bias = 0.;
    std::map<std::uint32_t, double> coef;
};

} // namespace

nn_plan make_nn_plan(const hy_program &p)
{
    nn_plan pl;
    const std::uint32_t n_eq = p.n_eq, n_uvars = p.n_uvars, n_ops = n_uvars - n_eq;
    try {
        if (n_ops == 0u || p.n_pars != 0u) {
            throw fail{"no operations / runtime parameters"};
        }
        const auto op_of = [&](std::uint32_t u) -> const hy_op & { return p.ops[u - n_eq]; };
        std::vector<char> visited(n_ops, 0);

        // ---- activations: tanh(u) with its hidden dependency square(tanh(u)) ----
        std::vector<char> is_base(n_uvars, 0); // state variables and activation outputs
        for (std::uint32_t s = 0; s < n_eq; ++s) {
            is_base[s] = 1;
        }
        for (std::uint32_t i = 0; i < n_ops; ++i) {
            const auto &op = p.ops[i];
            if (op.opcode == HY_OP_TANH) {
                const auto dep = op.c;
                if (dep < n_eq || op_of(dep).opcode != HY_OP_SQUARE || op_of(dep).a != n_eq + i) {
                    throw fail{"tanh without its squared hidden dependency"};
                }
                is_base[n_eq + i] = 1;
                visited[i] = 1;
                visited[dep - n_eq] = 1;
            }
        }

        // ---- linear forms ----
        // (Recursion depth = depth of the nested sums, a few levels.)
        const std::function<void(std::uint32_t, double, linear_form &)> expand = [&](std::uint32_t u, double scale,
                                                                                   linear_form &lf) {
            if (is_base[u]) {
                lf.coef[u] += scale;
                return;
            }
            const auto &op = op_of(u);
            visited[u - n_eq] = 1;
            switch (op.opcode) {
                case HY_OP_SUM:
                    for (std::uint32_t k = 0; k < op.b; ++k) {
                        const auto ref = p.args[op.a + k];
                        if (HY_REF_KIND(ref) == HY_REF_VAR) {
                            expand(HY_REF_IDX(ref), scale, lf);
                        } else if (HY_REF_KIND(ref) == HY_REF_NUM) {
                            lf.bias += scale * p.consts[HY_REF_IDX(ref)];
                        } else {
                            throw fail{"parameter inside a neuron"};
                        }
                    }
                    break;
                case HY_OP_MUL_NV:
                    expand(op.b, scale * p.consts[op.a], lf);
                    break;
                case HY_OP_NEG:
                    expand(op.a, -scale, lf);
                    break;
                // Weights of +-1 are folded into plain variables and negations, and the sums that hold them into
                // differences: x - y, x - b, b - x.
                case HY_OP_SUB_VV:
                    expand(op.a, scale, lf);
                    expand(op.b, -scale, lf);
                    break;
                case HY_OP_SUB_VN:
                    expand(op.a, scale, lf);
                    lf.bias -= scale * p.consts[op.b];
                    break;
                case HY_OP_SUB_NV:
                    lf.bias += scale * p.consts[op.a];
                    expand(op.b, -scale, lf);
                    break;
                default:
                    throw fail{"a neuron contains opcode " + std::to_string(op.opcode)};
            }
        };

        // Roots: the argument of every activation, and the right-hand side of every state variable.
        struct neuron {
            std::uint32_t u = 0;   // pre-activation u variable
            std::uint32_t out = 0; // activation output (hidden layers)
            int act = 0;
            linear_form lf;
            std::uint32_t level = 0;
        };
        std::vector<neuron> neurons;
        std::map<std::uint32_t, std::size_t> neuron_of_out; // activation output -> neuron
        for (std::uint32_t i = 0; i < n_ops; ++i) {
            if (p.ops[i].opcode == HY_OP_TANH) {
                neuron nr;
                nr.u = p.ops[i].a;
                nr.out = n_eq + i;
                nr.act = 1;
                if (is_base[nr.u]) {
                    throw fail{"activation applied directly to a state variable / activation"};
                }
                expand(nr.u, 1., nr.lf);
                neuron_of_out[nr.out] = neurons.size();
                neurons.push_back(std::move(nr));
            }
        }
        std::vector<std::size_t> out_neuron(n_eq);
        for (std::uint32_t s = 0; s < n_eq; ++s) {
            const auto ref = p.sv_defs[s];
            if (HY_REF_KIND(ref) != HY_REF_VAR || HY_REF_IDX(ref) < n_eq || is_base[HY_REF_IDX(ref)]) {
                throw fail{"a state variable's derivative is not an output neuron"};
            }
            const auto u = HY_REF_IDX(ref);
            std::size_t found = neurons.size();
            for (std::size_t k = 0; k < neurons.size(); ++k) {
                if (neurons[k].act == 0 && neurons[k].u == u) {
                    found = k;
                }
            }
            if (found == neurons.size()) {
                neuron nr;
                nr.u = u;
                nr.act = 0;
                expand(u, 1., nr.lf);
                neurons.push_back(std::move(nr));
            }
            out_neuron[s] = found;
        }
        for (std::uint32_t i = 0; i < n_ops; ++i) {
            if (!visited[i]) {
                throw fail{"operation outside of the network (u_" + std::to_string(n_eq + i) + ")"};
            }
        }

        // ---- levels: a neuron sits one level above its inputs ----
        for (bool changed = true; changed;) {
            changed = false;
            for (auto &nr : neurons) {
                std::uint32_t lvl = 1;
                for (const auto &[b, c] : nr.lf.coef) {
                    (void)c;
                    if (b >= n_eq) {
                        lvl = std::max(lvl, neurons[neuron_of_out.at(b)].level + 1u);
                    }
                }
                if (lvl != nr.level) {
                    nr.level = lvl;
                    changed = true;
                }
            }
        }
        std::uint32_t n_levels = 0;
        for (const auto &nr : neurons) {
            n_levels = std::max(n_levels, nr.level);
        }
        if (n_levels == 0u || n_levels > 8u) {
            throw fail{"unsupported depth"};
        }
        // ---- layers ----
        std::vector<std::vector<std::size_t>> by_level(n_levels + 1u);
        for (std::size_t k = 0; k < neurons.size(); ++k) {
            by_level[neurons[k].level].push_back(k);
        }
        std::vector<std::uint32_t> prev_outs; // activation outputs of the previous layer, in neuron order
        for (std::uint32_t s = 0; s < n_eq; ++s) {
            prev_outs.push_back(s);
        }
        for (std::uint32_t lv = 1; lv <= n_levels; ++lv) {
            const auto &ids = by_level[lv];
            if (ids.empty()) {
                throw fail{"empty layer"};
            }
            nn_layer L;
            L.n_in = static_cast<std::uint32_t>(prev_outs.size());
            L.n_out = static_cast<std::uint32_t>(ids.size());
            L.act = neurons[ids[0]].act;
            if ((L.act == 0) != (lv == n_levels)) {
                throw fail{"only the last layer may be linear, and it must be"};
            }
            L.w.assign(static_cast<std::size_t>(L.n_in) * L.n_out, 0.);
            L.bias.assign(L.n_out, 0.);
            std::map<std::uint32_t, std::uint32_t> col;
            for (std::uint32_t j = 0; j < L.n_in; ++j) {
                col[prev_outs[j]] = j;
            }
            std::vector<std::uint32_t> outs;
            for (std::uint32_t r = 0; r < L.n_out; ++r) {
                const auto &nr = neurons[ids[r]];
                if (nr.act != L.act) {
                    throw fail{"mixed activations in a layer"};
                }
                L.bias[r] = nr.lf.bias;
                L.u_out.push_back(nr.u);
                for (const auto &[b, c] : nr.lf.coef) {
                    const auto it = col.find(b);
                    if (it == col.end()) {
                        throw fail{"a neuron reads something else than the previous layer"};
                    }
                    L.w[static_cast<std::size_t>(r) * L.n_in + it->second] = c;
                }
                outs.push_back(nr.out);
            }
            pl.layers.push_back(std::move(L));
            prev_outs = std::move(outs);
        }
        // Output neurons -> state variables.
        const auto &last = by_level[n_levels];
        for (std::uint32_t s = 0; s < n_eq; ++s) {
            const auto it = std::find(last.begin(), last.end(), out_neuron[s]);
            if (it == last.end()) {
                throw fail{"a state variable derives from a hidden neuron"};
            }
            pl.out_of_sv.push_back(static_cast<std::uint32_t>(it - last.begin()));
        }
        pl.ok = true;
    } catch (const fail &f) {
        pl = nn_plan{};
        pl.why = f.why;
    } catch (const std::out_of_range &) {
        pl = nn_plan{};
        pl.why = "a neuron reads an activation that is not part of the network";
    }
    return pl;
}

} // namespace heyoka_b200::detail
