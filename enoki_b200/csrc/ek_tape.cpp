/*
 * ek_tape.cpp -- reverse/forward-mode tape runtime.
 *
 * Behavioural spec = src/autodiff/autodiff.cpp of the reference:
 *   Node/Edge/Special/Detail :44-192, append* :266-338, special edges :354-608,
 *   append_edge :610-643, ref counting :681-774, set_gradient :822-836,
 *   backward :838-910, forward :912-988, safe_mul/safe_fmadd :1191-1221.
 *
 * Re-designed for the GPU: instead of growing the evaluator trace by four nodes
 * per edge (the reference's CUDA branch), backward() levels the reachable sub-graph
 * and runs ONE adjoint kernel per level over materialised weights (ek_adjoint.cu).
 * Sources that need something the kernel does not do (special edges, size-1 sources
 * of wide edges -> hsum, pre-seeded gradients) take a generic path that records the
 * reference's exact op sequence through the evaluator (MUL_NZ / FMA_NZ / HSUM ...).
 * Per source, contributions are accumulated in descending target id -- the
 * reference's order -- so fp results match the CPU tape bit for bit.
 */
#include "ek_internal.h"
#include "ek_adjoint.h"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <sstream>
#include <unordered_set>

namespace {

enum SpecialKind { SP_GATHER, SP_SCATTER, SP_PSUM, SP_REVERSE };

struct Special {
    SpecialKind kind;
    uint32_t offset = 0, mask = 0;      /* evaluator variables (one ext ref each) */
    size_t size = 0;
    bool permute = false, scatter_add = false;
    ~Special() { if (offset) ek_dec_ref_ext(offset); if (mask) ek_dec_ref_ext(mask); }
};

struct TEdge {
    uint32_t source = 0;
    uint32_t weight = 0;                 /* evaluator variable (one ext ref) */
    Special *special = nullptr;
};

struct TNode {
    std::string label;
    uint32_t grad = 0;                   /* evaluator variable (one ext ref), 0 = empty */
    std::vector<TEdge> edges;            /* in-edges */
    std::vector<uint32_t> edges_rev;     /* targets of out-edges */
    uint32_t ref_ext = 0, ref_int = 0;
    uint32_t size = 0;
};

/* set of node ids with O(1) insert / membership; iteration is in ascending id order (what std::set gave the
   reference, autodiff.cpp:157) but sorted only once, when the sweep starts */
struct IdSet {
    std::vector<uint32_t> items;
    std::vector<uint8_t> mark;
    bool sorted = true;
    bool count(uint32_t k) const { return k < mark.size() && mark[k]; }
    void insert(uint32_t k) {
        if (k >= mark.size()) mark.resize((size_t) k + 1 + mark.size() / 2, 0);
        if (mark[k]) return;
        mark[k] = 1;
        if (!items.empty() && k < items.back()) sorted = false;
        items.push_back(k);
    }
    void clear() { for (uint32_t k : items) mark[k] = 0; items.clear(); sorted = true; }
    bool empty() const { return items.empty(); }
    const std::vector<uint32_t> &ordered() { if (!sorted) { std::sort(items.begin(), items.end()); sorted = true; } return items; }
};

struct Tape {
    ek_type vt = EK_FLOAT32;
    std::unordered_map<uint32_t, TNode> nodes;
    uint32_t node_counter = 1, node_counter_last = 1;
    std::vector<std::string> prefix;
    uint32_t *sg_index = nullptr;
    size_t sg_size = 0;
    bool sg_permute = false;
    uint32_t log_level = 0;
    bool graph_simplification = true, is_simplified = true;
    IdSet scheduled;
    /* staging for adjoint descriptors (persistent, grown on demand) */
    void *h_stage = nullptr, *d_stage = nullptr;
    size_t stage_bytes = 0;
    cudaEvent_t stage_done = nullptr;
};

Tape *g_tapes[2] = { nullptr, nullptr };

int simplify_graph(Tape &T);

/* autodiff.cpp:248-252: the tape simplifies itself right before every cuda_eval() */
void tape_eval_callback(void *p) {
    Tape *T = (Tape *) p;
    if (T->graph_simplification) simplify_graph(*T);
}

Tape *tape_of(ek_type t) {
    int i = t == EK_FLOAT64 ? 1 : 0;
    if (t == EK_FLOAT16) { ek_set_error("tape: Float16 is a storage format: the value type must be Float32 or Float64"); return nullptr; }
    if (t != EK_FLOAT32 && t != EK_FLOAT64) { ek_set_error("tape: value type must be Float32 or Float64"); return nullptr; }
    if (!g_tapes[i]) {
        g_tapes[i] = new Tape(); g_tapes[i]->vt = t;
        ek_register_callback(tape_eval_callback, g_tapes[i]);      /* autodiff.cpp:214-221 */
    }
    return g_tapes[i];
}

/* RAII equivalent of the reference's SimplificationLock (autodiff.cpp:194-205) */
struct SimplifyLock {
    Tape &T; bool saved;
    explicit SimplifyLock(Tape &t) : T(t), saved(t.graph_simplification) { T.graph_simplification = false; }
    ~SimplifyLock() { T.graph_simplification = saved; }
};

TNode *node(Tape &T, uint32_t idx) {
    auto it = T.nodes.find(idx);
    if (it == T.nodes.end()) { ek_set_error("autodiff: Detail::node(): Unknown index " + std::to_string(idx)); return nullptr; }   /* autodiff.cpp:164-169 */
    return &it->second;
}

/* ---- evaluator helpers ---- */
uint32_t v_literal(ek_type t, double value) {
    uint64_t bits;
    if (t == EK_FLOAT32) { float f = (float) value; uint32_t u; memcpy(&u, &f, 4); bits = u; }
    else memcpy(&bits, &value, 8);
    return ek_trace_append(t, EK_OP_LITERAL, 0, 0, 0, bits);
}
uint32_t v_op(ek_type t, ek_op op, uint32_t a, uint32_t b = 0, uint32_t c = 0, uint64_t imm = 0) {
    return ek_trace_append(t, op, a, b, c, imm);
}
void set_grad(TNode &n, uint32_t h /* takes ownership of one ext ref */) {
    if (n.grad) ek_dec_ref_ext(n.grad);
    n.grad = h;
}

void free_node(Tape &T, uint32_t idx);

void inc_ref_int(Tape &T, uint32_t idx, uint32_t from) {
    TNode *n = node(T, idx); if (!n) return;
    n->edges_rev.push_back(from);
    n->ref_int++;
}
void dec_ref_int(Tape &T, uint32_t idx, uint32_t from) {
    if (idx == 0) return;
    TNode *n = node(T, idx); if (!n) return;
    if (n->ref_int == 0) { fprintf(stderr, "autodiff: dec_ref_int(): Node %u has no internal references!\n", idx); exit(EXIT_FAILURE); }
    --n->ref_int;
    auto it = std::find(n->edges_rev.begin(), n->edges_rev.end(), from);
    if (it != n->edges_rev.end()) n->edges_rev.erase(it);
    if (n->ref_int == 0 && n->ref_ext == 0) free_node(T, idx);
}
void inc_ref_ext(Tape &T, uint32_t idx) {
    if (idx == 0) return;
    TNode *n = node(T, idx); if (n) n->ref_ext++;
}
void dec_ref_ext(Tape &T, uint32_t idx) {
    if (idx == 0) return;
    auto it = T.nodes.find(idx);
    if (it == T.nodes.end()) return;
    TNode &n = it->second;
    if (n.ref_ext == 0) { fprintf(stderr, "autodiff: dec_ref_ext(): Node %u has no external references!\n", idx); exit(EXIT_FAILURE); }
    --n.ref_ext;
    if (n.ref_int == 0 && n.ref_ext == 0) free_node(T, idx);
}
void release_edge(TEdge &e) {
    if (e.weight) { ek_dec_ref_ext(e.weight); e.weight = 0; }
    delete e.special; e.special = nullptr;
}
/* autodiff.cpp:759-774, iterative */
void free_node(Tape &T, uint32_t first) {
    std::vector<uint32_t> work { first };
    while (!work.empty()) {
        uint32_t idx = work.back(); work.pop_back();
        auto it = T.nodes.find(idx);
        if (it == T.nodes.end()) continue;
        TNode &n = it->second;
        if (n.ref_int != 0 || n.ref_ext != 0) continue;
        for (TEdge &e : n.edges) {
            if (e.source) {
                auto sit = T.nodes.find(e.source);
                if (sit != T.nodes.end()) {
                    TNode &s = sit->second;
                    if (s.ref_int > 0) --s.ref_int;
                    auto r = std::find(s.edges_rev.begin(), s.edges_rev.end(), idx);
                    if (r != s.edges_rev.end()) s.edges_rev.erase(r);
                    if (s.ref_int == 0 && s.ref_ext == 0) work.push_back(e.source);
                }
            }
            release_edge(e);
        }
        if (n.grad) ek_dec_ref_ext(n.grad);
        T.nodes.erase(it);
    }
}

uint32_t append_node(Tape &T, size_t size, const char *label) {
    uint32_t idx = T.node_counter++;
    TNode &n = T.nodes[idx];
    n.size = (uint32_t) size;
    n.label = label ? label : "";
    for (auto it = T.prefix.rbegin(); it != T.prefix.rend(); ++it) n.label = *it + '/' + n.label;
    n.ref_ext = 1;
    T.is_simplified = false;
    return idx;
}

int append_edge(Tape &T, uint32_t src, uint32_t dst, uint32_t weight) {
    if (src == 0) return 0;
    TNode *t = node(T, dst); if (!t) return -1;
    if (!node(T, src)) return -1;
    for (TEdge &e : t->edges) {
        if (e.source == src && !e.special) {           /* merge duplicate edges: autodiff.cpp:624-633 */
            uint32_t sum = v_op(T.vt, EK_OP_ADD, e.weight, weight);
            if (!sum) return -1;
            ek_dec_ref_ext(e.weight);
            e.weight = sum;
            return 0;
        }
    }
    TEdge e; e.source = src; e.weight = weight;
    ek_inc_ref_ext(weight);
    t->edges.push_back(e);
    inc_ref_int(T, src, dst);
    return 0;
}

void dfs(Tape &T, uint32_t root, bool backward, bool clear_grad) {
    /* autodiff.cpp:171-191, iterative */
    std::vector<uint32_t> stack { root };
    while (!stack.empty()) {
        uint32_t k = stack.back(); stack.pop_back();
        if (T.scheduled.count(k)) continue;
        TNode *n = node(T, k); if (!n) continue;
        T.scheduled.insert(k);
        if (clear_grad) set_grad(*n, 0);
        if (backward) { for (const TEdge &e : n->edges) if (e.source) stack.push_back(e.source); }
        else { for (uint32_t k2 : n->edges_rev) stack.push_back(k2); }
    }
}

/* broadcast a size-1 gradient to the node size (autodiff.cpp:851-861) */
int fix_grad_size(Tape &T, TNode &n) {
    if (!n.grad) return 0;
    size_t gs = ek_var_size(n.grad);
    if (gs == n.size) return 0;
    if (gs == 1) {
        uint32_t h = ek_var_set_size(n.grad, n.size, 1);
        if (!h) return -1;
        n.grad = h;
        return 0;
    }
    ek_set_error("backward(): gradient sizes don't match: expected " + std::to_string(n.size) + ", got " + std::to_string(gs));
    return -1;
}

/* literal value of a size-1 variable if it can be determined without evaluating it */
bool var_imm(uint32_t h, uint64_t &bits) {
    EkContext &ctx = ek_ctx();
    const EkVariable *v = &ctx.vars[h];
    if (v->op == EK_OP_MOV && v->data == nullptr && v->dep[0] >= EK_REG_RESERVED) v = &ctx.vars[v->dep[0]];   /* set_slices of a literal */
    if (v->op == EK_OP_LITERAL && v->data == nullptr) { bits = v->imm; return true; }
    return false;
}

/* ---- generic (trace-recorded) accumulation of one source, autodiff.cpp:863-888 + specials ---- */
int accumulate_generic(Tape &T, uint32_t sidx, TNode &s, const std::vector<std::pair<uint32_t, TEdge *>> &out) {
    for (auto &te : out) {
        TNode &t = *node(T, te.first);
        TEdge &e = *te.second;
        if (fix_grad_size(T, t) != 0) return -1;
        uint32_t g = t.grad;
        if (!g) continue;
        if (!e.special) {
            size_t ws = ek_var_size(e.weight), gs = ek_var_size(g);
            if (s.size == 1 && (ws != 1 || gs != 1)) {
                uint32_t m = v_op(T.vt, EK_OP_MUL_NZ, e.weight, g); if (!m) return -1;
                uint32_t h = v_op(T.vt, EK_OP_HSUM, m); ek_dec_ref_ext(m); if (!h) return -1;
                if (!s.grad) set_grad(s, h);
                else { uint32_t a = v_op(T.vt, EK_OP_ADD, s.grad, h); ek_dec_ref_ext(h); if (!a) return -1; set_grad(s, a); }
            } else {
                uint32_t r = s.grad ? v_op(T.vt, EK_OP_FMA_NZ, e.weight, g, s.grad) : v_op(T.vt, EK_OP_MUL_NZ, e.weight, g);
                if (!r) return -1;
                set_grad(s, r);
            }
            ek_ctx().stats.edge_adjoints += std::max<uint64_t>(std::max<uint64_t>(ws, gs), s.size);
        } else {
            const Special &sp = *e.special;
            switch (sp.kind) {
                case SP_GATHER: {              /* autodiff.cpp:384-398: scatter(_add) into a zero-initialised source grad */
                    size_t es = ek_type_size(T.vt);
                    if (!s.grad) {
                        void *p = ek_malloc(sp.size * es);
                        ek_fill(p, 1, 0, sp.size * es);
                        set_grad(s, ek_var_register(T.vt, sp.size, p, 1));
                    } else if (ek_var_size(s.grad) != sp.size) { ek_set_error("Internal error in Gather::backward()!"); return -1; }
                    if (ek_eval_var(s.grad) != 0) return -1;
                    if (ek_set_scatter_gather_operand(s.grad, 0) != 0) return -1;
                    uint32_t ptr = ek_var_register_ptr(ek_var_ptr(s.grad));
                    uint32_t h = v_op(sp.permute ? EK_UINT64 : T.vt, sp.permute ? EK_OP_SCATTER : EK_OP_SCATTER_ADD, ptr, sp.offset, sp.mask,
                                      ((uint64_t) es << 32) | g);
                    ek_dec_ref_ext(ptr);
                    ek_set_scatter_gather_operand(0, 0);
                    if (!h) return -1;
                    ek_var_mark_side_effect(h);
                    ek_var_mark_dirty(s.grad);
                } break;
                case SP_SCATTER: {             /* autodiff.cpp:553-571: gather (+ hsum for size-1 sources) */
                    if (ek_var_size(g) != sp.size) { ek_set_error("Internal error in Scatter::backward()!"); return -1; }
                    if (ek_set_scatter_gather_operand(g, 1) != 0) return -1;
                    uint32_t ptr = ek_var_register_ptr(ek_var_ptr(g));
                    uint32_t r = v_op(T.vt, EK_OP_GATHER, ptr, sp.offset, sp.mask, ek_type_size(T.vt));
                    ek_dec_ref_ext(ptr);
                    ek_set_scatter_gather_operand(0, 0);
                    if (!r) return -1;
                    if (s.size == 1 && ek_var_size(r) != 1) { uint32_t h = v_op(T.vt, EK_OP_HSUM, r); ek_dec_ref_ext(r); r = h; if (!r) return -1; }
                    else if (ek_var_size(r) == 1 && s.size != 1) { r = ek_var_set_size(r, s.size, 1); if (!r) return -1; }
                    if (!s.grad) set_grad(s, r);
                    else { uint32_t a = v_op(T.vt, EK_OP_ADD, s.grad, r); ek_dec_ref_ext(r); if (!a) return -1; set_grad(s, a); }
                } break;
                case SP_REVERSE: {             /* autodiff.cpp:442-452 */
                    if (ek_eval_var(g) != 0) return -1;
                    size_t n = ek_var_size(g), es = ek_type_size(T.vt);
                    void *p = ek_malloc(n * es);
                    ek_reverse(p, ek_var_ptr(g), es, n);
                    uint32_t r = ek_var_register(T.vt, n, p, 1);
                    if (!s.grad) set_grad(s, r);
                    else { uint32_t a = v_op(T.vt, EK_OP_ADD, s.grad, r); ek_dec_ref_ext(r); if (!a) return -1; set_grad(s, a); }
                } break;
                case SP_PSUM: {                /* autodiff.cpp:492-502: reverse(psum(reverse(g))) */
                    if (ek_eval_var(g) != 0) return -1;
                    size_t n = ek_var_size(g), es = ek_type_size(T.vt);
                    void *r1 = ek_malloc(n * es);
                    ek_reverse(r1, ek_var_ptr(g), es, n);
                    void *ps = ek_psum(T.vt, n, r1);
                    if (!ps) { ek_free(r1); return -1; }
                    ek_reverse(r1, ps, es, n);
                    ek_free(ps);
                    uint32_t r = ek_var_register(T.vt, n, r1, 1);
                    if (!s.grad) set_grad(s, r);
                    else { uint32_t a = v_op(T.vt, EK_OP_ADD, s.grad, r); ek_dec_ref_ext(r); if (!a) return -1; set_grad(s, a); }
                } break;
            }
        }
    }
    (void) sidx;
    return 0;
}

/* end-of-target bookkeeping, autodiff.cpp:884-898 */
void finalize_target(Tape &T, uint32_t tidx, bool free_graph) {
    auto it = T.nodes.find(tidx);
    if (it == T.nodes.end()) return;
    TNode &t = it->second;
    if (free_graph) {
        if (!t.edges.empty()) {
            std::vector<TEdge> edges;
            edges.swap(t.edges);
            set_grad(t, 0);
            for (TEdge &e : edges) { uint32_t src = e.source; release_edge(e); dec_ref_int(T, src, tidx); }
        }
        dec_ref_ext(T, tidx);
    } else {
        if (t.ref_int > 0) set_grad(t, 0);
    }
}

int backward_impl(Tape &T, bool free_graph) {
    EkContext &ctx = ek_ctx();
    std::vector<uint32_t> sched(T.scheduled.ordered());     /* ascending */
    if (sched.empty()) return 0;
    if (ek_init() != 0) return -1;
    if (free_graph) for (uint32_t idx : sched) inc_ref_ext(T, idx);
    const size_t es = ek_type_size(T.vt);
    const size_t S = sched.size();

    /* ---- one pass over the reachable sub-graph: node pointers, out-edge lists (sorted by
            descending target id because targets are visited in descending id), levels = longest
            distance from a root over out-edges ---- */
    struct SNode {
        TNode *n = nullptr;
        uint32_t level = 0, remaining = 0;
        int32_t block = -1;                                  /* level block that holds this node's adjoint */
    };
    typedef std::pair<uint32_t, TEdge *> OutEdge;            /* (target position, edge) */
    struct OutRange { OutEdge *b, *e; OutEdge *begin() const { return b; } OutEdge *end() const { return e; } size_t size() const { return (size_t) (e - b); } };
    /* adjoints of interior nodes of one level share ONE allocation (views into it); the block goes back
       to the allocator when the last of them has been consumed.  Leaves keep individual buffers: their
       gradients outlive backward(). */
    struct LevelBlock { void *base = nullptr; uint32_t pending = 0; };
    std::vector<SNode> sn(S);
    const uint32_t id_base = sched.front();
    std::vector<uint32_t> pos_of(sched.back() - id_base + 1, UINT32_MAX);
    for (size_t i = 0; i < S; ++i) { pos_of[sched[i] - id_base] = (uint32_t) i; sn[i].n = node(T, sched[i]); }
    uint32_t max_level = 0;
    bool need_eval = false;
    const bool any_dirty = !ctx.dirty.empty();
    size_t total_terms = 0;
    /* out-edge lists in CSR form (no per-node allocations): count, prefix-sum, fill */
    std::vector<uint32_t> out_start(S + 1, 0);
    auto src_pos = [&](const TEdge &e) -> uint32_t {
        if (e.source < id_base || e.source - id_base >= pos_of.size()) return UINT32_MAX;
        return pos_of[e.source - id_base];
    };
    for (size_t i = 0; i < S; ++i)
        for (TEdge &e : sn[i].n->edges) { uint32_t p = src_pos(e); if (p != UINT32_MAX) { ++out_start[p + 1]; ++total_terms; } }
    for (size_t i = 0; i < S; ++i) out_start[i + 1] += out_start[i];
    std::vector<OutEdge> out_items(total_terms);
    std::vector<uint32_t> cursor(out_start.begin(), out_start.end() - 1);
    for (size_t i = S; i-- > 0;) {
        TNode &t = *sn[i].n;
        sn[i].remaining = (uint32_t) t.edges.size();
        for (TEdge &e : t.edges) {
            uint32_t p = src_pos(e);
            if (p == UINT32_MAX) continue;
            sn[p].level = std::max(sn[p].level, sn[i].level + 1);
            max_level = std::max(max_level, sn[p].level);
            out_items[cursor[p]++] = OutEdge((uint32_t) i, &e);
            if (!e.special) {
                /* a dirty weight has pending side effects (the zeroing scatter of a scatter_combine edge):
                   the kernel must not read its buffer before they ran.  The flag sits on another cache line
                   than `data`, so it is only read while some variable is dirty at all. */
                const EkVariable &w = ctx.vars[e.weight];
                uint64_t bits;
                if ((w.data == nullptr && !var_imm(e.weight, bits)) || (any_dirty && w.dirty)) need_eval = true;
            }
        }
    }
    auto out_of = [&](uint32_t p) -> OutRange { return OutRange{ out_items.data() + out_start[p], out_items.data() + out_start[p + 1] }; };
    if (need_eval && ek_eval() != 0) return -1;           /* materialise all edge weights at once */

    std::vector<std::vector<uint32_t>> by_level(max_level + 1);
    for (size_t i = 0; i < S; ++i) by_level[sn[i].level].push_back((uint32_t) i);

    /* ---- descriptor staging: [jobs | terms | chunk_start] per level, one H2D copy each ---- */
    size_t need = S * (sizeof(EkAdjJob) + 4) + total_terms * sizeof(EkAdjTerm) + 64 * (max_level + 2);
    if (need > T.stage_bytes) {
        if (T.stage_done) { ek_cuda_check(cudaEventSynchronize(T.stage_done)); }
        if (T.h_stage) ek_host_free(T.h_stage);
        if (T.d_stage) ek_free(T.d_stage);
        T.stage_bytes = need + need / 2;
        T.h_stage = ek_host_malloc(T.stage_bytes);
        T.d_stage = ek_malloc(T.stage_bytes);
    }
    if (!T.stage_done) ek_cuda_check(cudaEventCreateWithFlags(&T.stage_done, cudaEventDisableTiming));
    else ek_cuda_check(cudaEventSynchronize(T.stage_done));   /* previous backward() has consumed the staging area */
    size_t stage_off = 0;

    /* roots / level 0: nothing to accumulate; leaves among them are finalised at once */
    std::vector<uint32_t> done, generic;
    uint8_t *hst = (uint8_t *) T.h_stage, *dst_dev = (uint8_t *) T.d_stage;
    std::vector<LevelBlock> blocks(max_level + 1);
    bool any_generic = false;
    /* (a gradient that the generic path leaves as an unevaluated trace may read views of several blocks) */
    auto finalize = [&](uint32_t p) {
        finalize_target(T, sched[p], free_graph);
        int32_t b = sn[p].block;
        if (b >= 0) {
            sn[p].block = -1;
            if (--blocks[b].pending == 0 && !any_generic && blocks[b].base) { ek_free(blocks[b].base); blocks[b].base = nullptr; }
        }
    };

    /* roots / level 0: nothing to accumulate; leaves among them are finalised at once */
    for (uint32_t p : by_level[0])
        if (sn[p].n->edges.empty()) finalize(p);

    /* Level launches are batched: the host builds the descriptors of consecutive levels back to back in the pinned
       staging area and flush() sends them with ONE copy followed by the launches, so the stream sees kernel after
       kernel instead of copy / kernel / copy ... (a few levels per batch, so that the GPU already works on the first
       levels while the host describes the next ones).  Anything that enqueues other work (generic path, ek_eval, an
       allocator trim) flushes first; the levels still execute in order. */
    struct PendingLaunch { size_t o_jobs, o_terms, o_chunks, end; uint32_t n_jobs, n_chunks; };
    struct Batch {
        std::vector<PendingLaunch> items;
        Tape *T; EkContext *ctx; uint8_t *hst, *dst_dev;
        void flush() {
            if (items.empty()) return;
            ek_cuda_check(cudaMemcpyAsync(dst_dev + items.front().o_jobs, hst + items.front().o_jobs,
                                          items.back().end - items.front().o_jobs, cudaMemcpyHostToDevice, ctx->stream));
            for (const PendingLaunch &pl : items) {
                unsigned grid = std::min<uint32_t>(pl.n_chunks, (uint32_t) ctx->num_sms * 8u);
                if (ctx->timing) ek_cuda_check(cudaEventRecord(ctx->ev_start, ctx->stream));
                ek_cuda_check(ek_launch_adjoint(T->vt == EK_FLOAT64, (const EkAdjJob *) (dst_dev + pl.o_jobs), (const EkAdjTerm *) (dst_dev + pl.o_terms),
                                                (const uint32_t *) (dst_dev + pl.o_chunks), pl.n_jobs, pl.n_chunks, grid, ctx->stream));
                if (ctx->timing) {
                    ek_cuda_check(cudaEventRecord(ctx->ev_stop, ctx->stream));
                    ek_cuda_check(cudaEventSynchronize(ctx->ev_stop));
                    float ms = 0; ek_cuda_check(cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop));
                    ctx->stats.last_kernel_ms = ms; ctx->stats.total_kernel_ms += ms;
                }
                ctx->stats.launches++; ctx->stats.adjoint_launches++;
            }
            items.clear();
        }
    } batch;
    batch.T = &T; batch.ctx = &ctx; batch.hst = hst; batch.dst_dev = dst_dev;
    struct HookGuard {
        EkContext &c;
        HookGuard(EkContext &c_, Batch *b) : c(c_) { c.pre_trim_hook = [](void *p) { ((Batch *) p)->flush(); }; c.pre_trim_arg = b; }
        ~HookGuard() { c.pre_trim_hook = nullptr; c.pre_trim_arg = nullptr; }
    } hook_guard(ctx, &batch);

    for (uint32_t L = 1; L <= max_level; ++L) {
        done.clear(); generic.clear();
        /* descriptors are written straight into the pinned staging area */
        const size_t n_src = by_level[L].size();
        size_t n_terms_lvl = 0;
        for (uint32_t p : by_level[L]) n_terms_lvl += out_of(p).size();
        size_t o_jobs = stage_off, o_terms = (o_jobs + n_src * sizeof(EkAdjJob) + 15) & ~(size_t) 15;
        size_t o_chunks = (o_terms + n_terms_lvl * sizeof(EkAdjTerm) + 15) & ~(size_t) 15;
        size_t end_max = (o_chunks + n_src * 4 + 15) & ~(size_t) 15;
        if (end_max > T.stage_bytes) { ek_set_error("backward(): internal error: staging overflow"); return -1; }
        EkAdjJob *jobs = (EkAdjJob *) (hst + o_jobs);
        EkAdjTerm *terms = (EkAdjTerm *) (hst + o_terms);
        uint32_t *chunk_start = (uint32_t *) (hst + o_chunks);
        uint32_t n_jobs = 0, n_terms = 0, n_chunks = 0;
        size_t block_bytes = 0, block_off = 0;
        for (uint32_t p : by_level[L])
            if (!sn[p].n->edges.empty()) block_bytes += ((size_t) sn[p].n->size * es + 511) & ~(size_t) 511;
        if (block_bytes) blocks[L].base = ek_malloc(block_bytes);

        for (uint32_t p : by_level[L]) {
            SNode &S_ = sn[p];
            TNode &s = *S_.n;
            /* classify */
            bool simple = s.grad == 0;
            for (auto &te : out_of(p)) {
                if (!simple) break;
                TNode &t = *sn[te.first].n;
                if (te.second->special) { simple = false; break; }
                const EkVariable &w = ctx.vars[te.second->weight];
                size_t ws = w.size, gs = t.grad ? ctx.vars[t.grad].size : 1;
                if (s.size == 1 && (ws != 1 || gs != 1)) { simple = false; break; }
                if ((ws != 1 && ws != s.size) || (gs != 1 && gs != s.size)) { simple = false; break; }
                if (t.grad) {
                    uint64_t bits;
                    const EkVariable &gv = ctx.vars[t.grad];
                    if ((gv.data == nullptr && !var_imm(t.grad, bits)) || gv.dirty) {
                        /* adjoint produced by the generic path: still an unevaluated trace, or a buffer with
                           pending scatter_add side effects (gather edges) */
                        batch.flush();
                        if (ek_eval() != 0) return -1;
                    }
                }
            }
            if (!simple) { generic.push_back(p); any_generic = true; continue; }

            EkAdjJob job;
            job.first_term = n_terms; job.n_terms = 0; job.size = s.size; job.aligned = 1;
            for (auto &te : out_of(p)) {
                TNode &t = *sn[te.first].n;
                if (!t.grad) continue;                      /* empty adjoint contributes nothing */
                EkAdjTerm &term = terms[n_terms]; term.pad = 0;
                uint32_t wk, gk; uint64_t bits;
                const EkVariable &w = ctx.vars[te.second->weight];
                if (w.data != nullptr) { wk = w.size == 1 ? EK_ADJ_SCALAR : EK_ADJ_ARRAY; term.w = (uint64_t) (uintptr_t) w.data; }
                else if (var_imm(te.second->weight, bits)) { wk = EK_ADJ_IMM; term.w = bits; }
                else { ek_set_error("backward(): internal error: edge weight not materialised"); return -1; }
                const EkVariable &g = ctx.vars[t.grad];
                if (g.data != nullptr) { gk = g.size == 1 ? EK_ADJ_SCALAR : EK_ADJ_ARRAY; term.g = (uint64_t) (uintptr_t) g.data; }
                else if (var_imm(t.grad, bits)) { gk = EK_ADJ_IMM; term.g = bits; }
                else { ek_set_error("backward(): internal error: target adjoint not materialised"); return -1; }
                if ((wk == EK_ADJ_ARRAY && (term.w & 15u)) || (gk == EK_ADJ_ARRAY && (term.g & 15u))) job.aligned = 0;
                term.flags = wk | (gk << 2);
                ++n_terms; job.n_terms++;
            }
            ctx.stats.edge_adjoints += (uint64_t) job.n_terms * s.size;
            if (job.n_terms > 0) {
                void *dst;
                if (!s.edges.empty()) {                        /* interior node: view into the level block */
                    dst = (uint8_t *) blocks[L].base + block_off;
                    block_off += ((size_t) s.size * es + 511) & ~(size_t) 511;
                    S_.block = (int32_t) L; blocks[L].pending++;
                    set_grad(s, ek_var_register(T.vt, s.size, dst, 0));
                } else {                                       /* leaf: its gradient outlives backward() */
                    dst = ek_malloc((size_t) s.size * es);
                    set_grad(s, ek_var_register(T.vt, s.size, dst, 1));
                }
                job.dst = (uint64_t) (uintptr_t) dst;
                chunk_start[n_jobs] = n_chunks;
                n_chunks += (s.size + EK_ADJ_CHUNK - 1) / EK_ADJ_CHUNK;
                jobs[n_jobs++] = job;
            }
            done.push_back(p);
        }

        if (n_jobs) {
            size_t end = (o_chunks + (size_t) n_jobs * 4 + 15) & ~(size_t) 15;
            batch.items.push_back({ o_jobs, o_terms, o_chunks, end, n_jobs, n_chunks });
            stage_off = end;
        }
        /* small batches keep the GPU busy while the host prepares the following levels */
        if (!generic.empty() || ctx.timing || batch.items.size() >= (L <= 2 ? 1u : 6u)) batch.flush();

        /* generic sources of this level (special edges, hsum into scalars, pre-seeded grads) */
        for (uint32_t p : generic) {
            std::vector<std::pair<uint32_t, TEdge *>> out;
            out.reserve(out_of(p).size());
            for (auto &te : out_of(p)) out.emplace_back(sched[te.first], te.second);
            if (accumulate_generic(T, sched[p], *sn[p].n, out) != 0) return -1;
            done.push_back(p);
        }

        /* bookkeeping: every processed source has consumed one in-edge of each of its targets */
        for (uint32_t p : done) {
            for (auto &te : out_of(p)) {
                SNode &tn = sn[te.first];
                if (tn.remaining > 0 && --tn.remaining == 0) finalize(te.first);
            }
            /* a source without in-edges (leaf) is complete now */
            if (sn[p].remaining == 0 && sn[p].n->edges.empty()) finalize(p);
        }
        if (blocks[L].base && blocks[L].pending == 0 && !any_generic) { ek_free(blocks[L].base); blocks[L].base = nullptr; }
    }
    batch.flush();
    ek_cuda_check(cudaEventRecord(T.stage_done, ctx.stream));
    /* blocks that could not be released early (the generic path may hold unevaluated traces that read
       adjoint views): evaluate, then release */
    bool left = false;
    for (auto &b : blocks) left |= b.base != nullptr;
    if (left) {
        if (any_generic && ek_eval() != 0) return -1;
        for (auto &b : blocks) if (b.base) { ek_free(b.base); b.base = nullptr; }
    }

    if (T.log_level >= 1)
        fprintf(stderr, "autodiff: backward(): processed %zu/%u nodes.\n", S, T.node_counter - T.node_counter_last);
    if (free_graph) T.node_counter_last = T.node_counter;
    T.scheduled.clear();
    return 0;
}

/* forward mode, autodiff.cpp:912-988 (recorded through the evaluator) */
int forward_impl(Tape &T, bool free_graph) {
    std::vector<uint32_t> sched(T.scheduled.ordered());
    if (free_graph) for (uint32_t idx : sched) inc_ref_ext(T, idx);
    for (uint32_t sidx : sched) {
        auto sit = T.nodes.find(sidx);
        if (sit == T.nodes.end()) continue;
        TNode &s = sit->second;
        if (s.size == 1 && s.grad && ek_var_size(s.grad) > 1) {
            uint32_t h = v_op(T.vt, EK_OP_HSUM, s.grad); if (!h) return -1; set_grad(s, h);
        }
        std::vector<uint32_t> targets = s.edges_rev;
        for (uint32_t tidx : targets) {
            TNode *tp = node(T, tidx); if (!tp) return -1;
            TNode &t = *tp;
            TEdge *e = nullptr;
            for (TEdge &x : t.edges) if (x.source == sidx) { e = &x; break; }
            if (!e) { ek_set_error("forward(): invalid graph structure!"); return -1; }
            if (s.grad) {
                if (!e->special) {
                    size_t ws = ek_var_size(e->weight), gs = ek_var_size(s.grad);
                    if (t.size == 1 && (ws != 1 || gs != 1)) {
                        uint32_t m = v_op(T.vt, EK_OP_MUL_NZ, e->weight, s.grad); if (!m) return -1;
                        uint32_t h = v_op(T.vt, EK_OP_HSUM, m); ek_dec_ref_ext(m); if (!h) return -1;
                        if (!t.grad) set_grad(t, h);
                        else { uint32_t a = v_op(T.vt, EK_OP_ADD, t.grad, h); ek_dec_ref_ext(h); if (!a) return -1; set_grad(t, a); }
                    } else {
                        uint32_t r = t.grad ? v_op(T.vt, EK_OP_FMA_NZ, e->weight, s.grad, t.grad) : v_op(T.vt, EK_OP_MUL_NZ, e->weight, s.grad);
                        if (!r) return -1;
                        set_grad(t, r);
                    }
                } else {
                    const Special &sp = *e->special;
                    uint32_t g = s.grad;
                    switch (sp.kind) {
                        case SP_GATHER: {          /* autodiff.cpp:367-382 */
                            if (ek_var_size(g) != sp.size) { ek_set_error("Internal error in Gather::forward()!"); return -1; }
                            if (ek_set_scatter_gather_operand(g, 1) != 0) return -1;
                            uint32_t ptr = ek_var_register_ptr(ek_var_ptr(g));
                            uint32_t r = v_op(T.vt, EK_OP_GATHER, ptr, sp.offset, sp.mask, ek_type_size(T.vt));
                            ek_dec_ref_ext(ptr);
                            ek_set_scatter_gather_operand(0, 0);
                            if (!r) return -1;
                            if (!t.grad) set_grad(t, r);
                            else { uint32_t a = v_op(T.vt, EK_OP_ADD, t.grad, r); ek_dec_ref_ext(r); if (!a) return -1; set_grad(t, a); }
                        } break;
                        case SP_SCATTER: {         /* autodiff.cpp:536-551 */
                            size_t es = ek_type_size(T.vt);
                            if (!t.grad) {
                                void *p = ek_malloc(sp.size * es);
                                ek_fill(p, 1, 0, sp.size * es);
                                set_grad(t, ek_var_register(T.vt, sp.size, p, 1));
                            } else if (ek_var_size(t.grad) != sp.size) { ek_set_error("Internal error in Scatter::forward()!"); return -1; }
                            if (ek_eval_var(t.grad) != 0) return -1;
                            if (ek_set_scatter_gather_operand(t.grad, 0) != 0) return -1;
                            uint32_t ptr = ek_var_register_ptr(ek_var_ptr(t.grad));
                            uint32_t h = v_op(sp.scatter_add ? T.vt : EK_UINT64, sp.scatter_add ? EK_OP_SCATTER_ADD : EK_OP_SCATTER, ptr, sp.offset, sp.mask,
                                              ((uint64_t) es << 32) | g);
                            ek_dec_ref_ext(ptr);
                            ek_set_scatter_gather_operand(0, 0);
                            if (!h) return -1;
                            ek_var_mark_side_effect(h);
                            ek_var_mark_dirty(t.grad);
                        } break;
                        case SP_REVERSE:           /* autodiff.cpp:430-440 */
                        case SP_PSUM: {            /* autodiff.cpp:480-490 */
                            if (ek_eval_var(g) != 0) return -1;
                            size_t n = ek_var_size(g), es = ek_type_size(T.vt);
                            void *p;
                            if (sp.kind == SP_PSUM) {
                                p = ek_psum(T.vt, n, ek_var_ptr(g));
                                if (!p) return -1;
                            } else {
                                p = ek_malloc(n * es);
                                ek_reverse(p, ek_var_ptr(g), es, n);
                            }
                            uint32_t r = ek_var_register(T.vt, n, p, 1);
                            if (!t.grad) set_grad(t, r);
                            else { uint32_t a = v_op(T.vt, EK_OP_ADD, t.grad, r); ek_dec_ref_ext(r); if (!a) return -1; set_grad(t, a); }
                        } break;
                    }
                }
            }
            if (fix_grad_size(T, t) != 0) return -1;
        }
        if (s.ref_int > 0) set_grad(s, 0);
        if (free_graph) {
            std::vector<uint32_t> rev = s.edges_rev;
            for (uint32_t tidx : rev) {
                TNode *tp = node(T, tidx); if (!tp) continue;
                for (auto it = tp->edges.begin(); it != tp->edges.end(); ++it)
                    if (it->source == sidx) { release_edge(*it); tp->edges.erase(it); break; }
                dec_ref_int(T, sidx, tidx);
            }
            dec_ref_ext(T, sidx);
        }
    }
    if (free_graph) T.node_counter_last = T.node_counter;
    T.scheduled.clear();
    return 0;
}

/* Greedy vertex elimination, behavioural spec autodiff.cpp:990-1074 (+ append_edge_prod :645-679):
   repeatedly collapse the interior node with the smallest in-degree x out-degree product (while that
   cost is <= 10): every (in-edge, out-edge) pair becomes one edge whose weight is the zero-guarded
   product of the two weights (added to an existing parallel edge with a zero-guarded fma).  Nodes
   touching special edges, and size-1 nodes fed by wide nodes, are left alone.  The new weights are
   ordinary trace expressions: they are fused into the next sweep and the collapsed node's own weight
   arrays are never materialised. */
int simplify_graph(Tape &T) {
    if (T.is_simplified) return 0;
    SimplifyLock lock(T);
    const uint32_t max_cost = 10;                       /* ENOKI_AUTODIFF_MAX_SIMPLIFICATION_COST */
    auto score = [](const TNode &n) { return (uint32_t) (n.edges.size() * n.edges_rev.size()); };
    std::set<std::pair<uint32_t, uint32_t>> todo;
    for (auto &kv : T.nodes) todo.emplace(score(kv.second), kv.first);
    std::vector<std::pair<uint32_t, uint32_t>> update;

    while (!todo.empty()) {
        auto it = todo.begin();
        uint32_t sc = it->first, index = it->second;
        todo.erase(it);
        auto nit = T.nodes.find(index);
        if (nit == T.nodes.end()) continue;
        TNode &n = nit->second;
        if (n.edges.empty() || n.edges_rev.empty()) continue;           /* collapse_allowed() */
        if (sc > max_cost) break;

        update.clear();
        bool skip = false;
        for (uint32_t k : n.edges_rev) {
            TNode *c = node(T, k); if (!c) return -1;
            for (const TEdge &e : c->edges) if (e.source == index && e.special) skip = true;
            update.emplace_back(score(*c), k);
        }
        for (const TEdge &e : n.edges) {
            TNode *src = node(T, e.source); if (!src) return -1;
            update.emplace_back(score(*src), e.source);
            if ((n.size == 1 && src->size != n.size) || e.special) skip = true;
        }
        if (skip) continue;

        std::vector<uint32_t> consumers = n.edges_rev;
        for (uint32_t other : consumers) {
            TNode &o = *node(T, other);
            /* detach the edge index -> other */
            TEdge edge1;
            bool found = false;
            for (auto eit = o.edges.begin(); eit != o.edges.end(); ++eit)
                if (eit->source == index && !eit->special) { edge1 = *eit; o.edges.erase(eit); found = true; break; }
            if (!found) { ek_set_error("simplify_graph(): internal error -- edge not found"); return -1; }
            for (const TEdge &edge2 : n.edges) {
                /* append_edge_prod(edge2.source, other, edge1.weight, edge2.weight) */
                TEdge *ex = nullptr;
                for (TEdge &e : o.edges) if (e.source == edge2.source && !e.special) { ex = &e; break; }
                if (ex) {
                    uint32_t w = v_op(T.vt, EK_OP_FMA_NZ, edge1.weight, edge2.weight, ex->weight);
                    if (!w) return -1;
                    ek_dec_ref_ext(ex->weight);
                    ex->weight = w;
                } else {
                    uint32_t w = v_op(T.vt, EK_OP_MUL_NZ, edge1.weight, edge2.weight);
                    if (!w) return -1;
                    TEdge ne; ne.source = edge2.source; ne.weight = w;      /* takes the ext ref of w */
                    o.edges.push_back(ne);
                    inc_ref_int(T, edge2.source, other);
                }
            }
            release_edge(edge1);
            dec_ref_int(T, index, other);          /* may free `index` (and cascade) once its last consumer is gone */
        }

        for (auto &u : update) {
            auto f = todo.find(u);
            if (f == todo.end()) continue;
            auto un = T.nodes.find(u.second);
            if (un == T.nodes.end()) { todo.erase(f); continue; }
            uint32_t ns = score(un->second);
            if (ns != u.first) { todo.erase(f); todo.emplace(ns, u.second); }
        }
    }
    T.is_simplified = true;
    return 0;
}

} // namespace

extern "C" {

uint32_t ek_tape_append_node(ek_type t, size_t size, const char *label) {
    Tape *T = tape_of(t); if (!T) return 0;
    return append_node(*T, size, label);
}

uint32_t ek_tape_append_leaf(ek_type t, size_t size) {
    Tape *T = tape_of(t); if (!T) return 0;
    uint32_t idx = append_node(*T, size, "'unnamed'");
    /* autodiff.cpp:331-338: leaf gets a zero gradient */
    TNode &n = T->nodes[idx];
    uint32_t z = v_literal(t, 0.0);
    if (size != 1) z = ek_var_set_size(z, size, 1);
    set_grad(n, z);
    return idx;
}

int ek_tape_append_edge(ek_type t, uint32_t src, uint32_t dst, uint32_t weight) {
    Tape *T = tape_of(t); if (!T) return -1;
    return append_edge(*T, src, dst, weight);
}

uint32_t ek_tape_append(ek_type t, const char *label, size_t size, uint32_t n_in,
                        const uint32_t *in, const uint32_t *weights) {
    Tape *T = tape_of(t); if (!T) return 0;
    bool any = false;
    for (uint32_t i = 0; i < n_in; ++i) any |= in[i] != 0;
    if (!any) return 0;                                   /* autodiff.cpp:268-269 */
    uint32_t idx = append_node(*T, size, label);
    for (uint32_t i = 0; i < n_in; ++i)
        if (append_edge(*T, in[i], idx, weights[i]) != 0) return 0;
    return idx;
}

uint32_t ek_tape_append_gather(ek_type t, uint32_t offset_var, uint32_t mask_var) {
    Tape *T = tape_of(t); if (!T) return 0;
    if (T->sg_index == nullptr || *T->sg_index == 0) return 0;
    uint32_t source = *T->sg_index;
    Special *sp = new Special();
    sp->kind = SP_GATHER; sp->offset = offset_var; sp->mask = mask_var;
    ek_inc_ref_ext(offset_var); ek_inc_ref_ext(mask_var);
    sp->size = T->sg_size; sp->permute = T->sg_permute;
    uint32_t target = append_node(*T, ek_var_size(offset_var), "gather");
    TEdge e; e.source = source; e.special = sp;
    T->nodes[target].edges.push_back(e);
    inc_ref_int(*T, source, target);
    return target;
}

int ek_tape_append_scatter(ek_type t, uint32_t source, uint32_t offset_var, uint32_t mask_var, int scatter_add) {
    Tape *T = tape_of(t); if (!T) return -1;
    if (T->sg_index == nullptr || source == 0) return 0;
    SimplifyLock lock(*T);                                  /* autodiff.cpp:526 */
    uint32_t target_orig = *T->sg_index;
    Special *sp = new Special();
    sp->kind = SP_SCATTER; sp->offset = offset_var; sp->mask = mask_var;
    ek_inc_ref_ext(offset_var); ek_inc_ref_ext(mask_var);
    sp->size = T->sg_size; sp->scatter_add = scatter_add != 0;
    uint32_t target_new = append_node(*T, T->sg_size, scatter_add ? "scatter_add" : "scatter");
    TEdge e; e.source = source; e.special = sp;
    T->nodes[target_new].edges.push_back(e);
    inc_ref_int(*T, source, target_new);
    if (target_orig != 0) {
        uint32_t sa_node = target_new;
        uint32_t one = v_literal(t, 1.0), weight;
        if (!scatter_add && !T->sg_permute) {
            /* weight zeroes the slots that were overwritten (autodiff.cpp:588-592) */
            size_t es = ek_type_size(t);
            void *p = ek_malloc(T->sg_size * es);
            uint64_t one_bits = ek_ctx().vars[one].imm;
            ek_fill(p, es, one_bits, T->sg_size);
            weight = ek_var_register(t, T->sg_size, p, 1);
            uint32_t zero = v_literal(t, 0.0);
            ek_set_scatter_gather_operand(weight, 0);
            uint32_t ptr = ek_var_register_ptr(p);
            uint32_t h = v_op(EK_UINT64, EK_OP_SCATTER, ptr, offset_var, mask_var, ((uint64_t) es << 32) | zero);
            ek_dec_ref_ext(ptr); ek_dec_ref_ext(zero);
            ek_set_scatter_gather_operand(0, 0);
            if (!h) return -1;
            ek_var_mark_side_effect(h);
            ek_var_mark_dirty(weight);
        } else {
            weight = one; ek_inc_ref_ext(one);
        }
        uint32_t in[2] = { target_new, target_orig }, w[2] = { one, weight };
        target_new = ek_tape_append(t, "scatter_combine", T->sg_size, 2, in, w);
        ek_dec_ref_ext(one); ek_dec_ref_ext(weight);
        dec_ref_ext(*T, sa_node);
        dec_ref_ext(*T, target_orig);
    }
    *T->sg_index = target_new;
    return 0;
}

uint32_t ek_tape_append_psum(ek_type t, uint32_t src) {
    Tape *T = tape_of(t); if (!T || src == 0) return 0;
    TNode *s = node(*T, src); if (!s) return 0;
    Special *sp = new Special(); sp->kind = SP_PSUM;
    uint32_t target = append_node(*T, s->size, "psum");
    TEdge e; e.source = src; e.special = sp;
    T->nodes[target].edges.push_back(e);
    inc_ref_int(*T, src, target);
    return target;
}

uint32_t ek_tape_append_reverse(ek_type t, uint32_t src) {
    Tape *T = tape_of(t); if (!T || src == 0) return 0;
    TNode *s = node(*T, src); if (!s) return 0;
    Special *sp = new Special(); sp->kind = SP_REVERSE;
    uint32_t target = append_node(*T, s->size, "reverse");
    TEdge e; e.source = src; e.special = sp;
    T->nodes[target].edges.push_back(e);
    inc_ref_int(*T, src, target);
    return target;
}

void ek_tape_inc_ref_ext(ek_type t, uint32_t index) { Tape *T = tape_of(t); if (T) inc_ref_ext(*T, index); }
void ek_tape_dec_ref_ext(ek_type t, uint32_t index) { Tape *T = tape_of(t); if (T) dec_ref_ext(*T, index); }

int ek_tape_set_scatter_gather_operand(ek_type t, uint32_t *index, size_t size, int permute) {
    Tape *T = tape_of(t); if (!T) return -1;
    if (index != nullptr && T->sg_index != nullptr) {
        ek_set_error("set_scatter_gather_operand(): attempted to override an existing operand!");   /* autodiff.cpp:788-790 */
        return -1;
    }
    T->sg_index = index; T->sg_size = size; T->sg_permute = permute != 0;
    return 0;
}

int ek_tape_set_gradient(ek_type t, uint32_t index, uint32_t value_var, int backward) {
    Tape *T = tape_of(t); if (!T) return -1;
    if (index == 0) {
        ek_set_error("set_gradient(): no gradients are associated with this variable (a prior call to requires_gradient() is required.) ");
        return -1;
    }
    if (!node(*T, index)) return -1;
    dfs(*T, index, backward != 0, true);
    TNode &n = *node(*T, index);
    ek_inc_ref_ext(value_var);
    set_grad(n, value_var);
    if (n.size > 1 && ek_var_size(n.grad) == 1) return fix_grad_size(*T, n);
    return 0;
}

int ek_tape_backward_static(ek_type t, int free_graph) {
    Tape *T = tape_of(t); if (!T) return -1;
    SimplifyLock lock(*T);
    int rc = backward_impl(*T, free_graph != 0);
    if (rc != 0) T->scheduled.clear();
    return rc;
}

int ek_tape_forward_static(ek_type t, int free_graph) {
    Tape *T = tape_of(t); if (!T) return -1;
    SimplifyLock lock(*T);
    int rc = forward_impl(*T, free_graph != 0);
    if (rc != 0) T->scheduled.clear();
    return rc;
}

int ek_tape_backward(ek_type t, uint32_t index, int free_graph) {
    Tape *T = tape_of(t); if (!T) return -1;
    SimplifyLock lock(*T);                                  /* autodiff.cpp:808 */
    uint32_t one = v_literal(t, 1.0);
    int rc = ek_tape_set_gradient(t, index, one, 1);
    ek_dec_ref_ext(one);
    if (rc != 0) return rc;
    return ek_tape_backward_static(t, free_graph);
}

int ek_tape_forward(ek_type t, uint32_t index, int free_graph) {
    Tape *T = tape_of(t); if (!T) return -1;
    SimplifyLock lock(*T);                                  /* autodiff.cpp:817 */
    uint32_t one = v_literal(t, 1.0);
    int rc = ek_tape_set_gradient(t, index, one, 0);
    ek_dec_ref_ext(one);
    if (rc != 0) return rc;
    return ek_tape_forward_static(t, free_graph);
}

uint32_t ek_tape_gradient(ek_type t, uint32_t index) {
    Tape *T = tape_of(t); if (!T) return 0;
    if (index == 0) {
        ek_set_error("No gradient was computed for this variable! (a call to requires_gradient() is necessary.)");   /* autodiff.cpp:797-800 */
        return 0;
    }
    TNode *n = node(*T, index); if (!n) return 0;
    ek_set_error("");
    return n->grad;
}

int ek_tape_set_label(ek_type t, uint32_t index, const char *label) {
    Tape *T = tape_of(t); if (!T) return -1;
    if (index == 0) return 0;
    TNode *n = node(*T, index); if (!n) return -1;
    n->label = "'" + std::string(label) + "'";
    if (n->grad) ek_var_set_label(n->grad, (std::string(label) + ".grad").c_str());
    return 0;
}

void ek_tape_push_prefix(ek_type t, const char *prefix) { Tape *T = tape_of(t); if (T) T->prefix.push_back(prefix); }
int ek_tape_pop_prefix(ek_type t) {
    Tape *T = tape_of(t); if (!T) return -1;
    if (T->prefix.empty()) { ek_set_error("pop_prefix(): prefix list is already empty!"); return -1; }
    T->prefix.pop_back();
    return 0;
}
void ek_tape_set_log_level(ek_type t, uint32_t level) { Tape *T = tape_of(t); if (T) T->log_level = level; }
void ek_tape_set_graph_simplification(ek_type t, int enable) { Tape *T = tape_of(t); if (T) T->graph_simplification = enable != 0; }

int ek_tape_simplify(ek_type t) {
    Tape *T = tape_of(t); if (!T) return -1;
    return simplify_graph(*T);
}

char *ek_tape_graphviz(ek_type t, size_t n, const uint32_t *indices) {
    Tape *T = tape_of(t); if (!T) return nullptr;
    /* autodiff.cpp:1076-1163 */
    std::ostringstream oss;
    oss << "digraph {\n  rankdir=BT;\n  graph [dpi=50];\n  node [shape=record fontname=Consolas];\n  edge [fontname=Consolas];\n";
    std::set<uint32_t> seen; std::vector<uint32_t> stack(indices, indices + n);
    while (!stack.empty()) {
        uint32_t k = stack.back(); stack.pop_back();
        if (k == 0 || seen.count(k)) continue;
        auto it = T->nodes.find(k); if (it == T->nodes.end()) continue;
        seen.insert(k);
        const TNode &nd = it->second;
        oss << "  " << k << " [label=\"" << nd.label << (nd.size == 1 ? " [s]" : "") << "\\n#" << k << " [E/I: " << nd.ref_ext << "/" << nd.ref_int << "]\""
            << (nd.edges.empty() ? " fillcolor=salmon style=filled" : "") << "];\n";
        for (const TEdge &e : nd.edges) {
            oss << "  " << k << " -> " << e.source << (e.special ? " [color=red]" : "") << ";\n";
            stack.push_back(e.source);
        }
    }
    oss << "}";
    return strdup(oss.str().c_str());
}

char *ek_tape_whos(ek_type t) {
    Tape *T = tape_of(t); if (!T) return nullptr;
    std::ostringstream oss;
    oss << "\n  ID        E/I Refs   Size        Label\n  ========================================\n";
    std::vector<uint32_t> ids;
    for (auto &kv : T->nodes) ids.push_back(kv.first);
    std::sort(ids.begin(), ids.end());
    for (uint32_t id : ids) {
        const TNode &n = T->nodes[id];
        char line[256];
        snprintf(line, sizeof(line), "  %-9u %u / %-6u %-11u %s\n", id, n.ref_ext, n.ref_int, n.size, n.label.c_str());
        oss << line;
    }
    oss << "  ========================================\n";
    return strdup(oss.str().c_str());
}

size_t ek_tape_node_count(ek_type t) { Tape *T = tape_of(t); return T ? T->nodes.size() : 0; }

void ek_tape_clear(ek_type t) {
    int i = t == EK_FLOAT64 ? 1 : 0;
    Tape *T = g_tapes[i];
    if (!T) return;
    std::vector<uint32_t> ids;
    for (auto &kv : T->nodes) ids.push_back(kv.first);
    for (uint32_t id : ids) {
        auto it = T->nodes.find(id);
        if (it == T->nodes.end()) continue;
        for (TEdge &e : it->second.edges) release_edge(e);
        if (it->second.grad) ek_dec_ref_ext(it->second.grad);
    }
    T->nodes.clear();
    T->scheduled.clear();
    T->sg_index = nullptr;
}

/* host-only test aid: evaluator handle of the weight of edge src -> dst (0 if there is no such ordinary edge); lets the
   CPU test-suite execute the fused weight products simplify_graph() records (tests/ek_emulator.py) */
EK_API uint32_t ek_debug_tape_edge_weight(ek_type t, uint32_t src, uint32_t dst) {
    Tape *T = tape_of(t); if (!T) return 0;
    auto it = T->nodes.find(dst);
    if (it == T->nodes.end()) return 0;
    for (const TEdge &e : it->second.edges)
        if (e.source == src && !e.special) return e.weight;
    return 0;
}

} /* extern "C" */
