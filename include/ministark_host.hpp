// ministark_host.hpp — C++17 host side of the prover above the C ABI (include/ministark_b200.h).
//
// The reference's host code is compiled Rust; cargo / rustc are not in this image, so the host layer that a Rust
// maintainer would write against the extern "C" boundary is mirrored here in C++ (header-only), next to the Python
// mirror in ministark_b200/ that the tests drive:
//
//     field helpers (canonical integers)         ark-ff Fp / CubicExtField semantics used on the host
//     Sha256, PublicCoin                         src/hash.rs:58-100, src/random.rs:91-196
//     ProofOptions, MerkleView, LayerProof, FriProof, Queries, Proof + wire format
//                                                src/lib.rs:86-132, src/merkle.rs:71-80, src/fri.rs:71-125,
//                                                src/trace.rs:37-66, src/proof.rs:43-66
//     Graph / Expr, degree rules, Air            src/expression.rs, src/constraints.rs:404-455, src/air.rs:50-82,142-247
//     compile_program / Program::bind            the fused evaluator's instruction stream (csrc/eval.cu), the same
//                                                algorithm as ministark_b200/expr.py
//
// Everything in this header is pure host logic and is tested on the CPU (tests/test_cpp_host.py drives
// tests/cpp/host_test.cpp and compares with the Python mirror / a big-integer interpreter of the emitted programs).
// The GPU-calling driver built on it lives in ministark_prover.hpp.
#pragma once
#include <algorithm>
#include <array>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <set>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

namespace mshost {

using u8 = uint8_t;
using u32 = uint32_t;
using u64 = uint64_t;
using u128 = unsigned __int128;
using Bytes = std::vector<u8>;

// ------------------------------------------------------------------------------------------------ field (canonical)
constexpr u64 P = 0xFFFFFFFF00000001ULL;
inline u64 addm(u64 a, u64 b) { return (u64)(((u128)a + b) % P); }
inline u64 subm(u64 a, u64 b) { return a >= b ? a - b : a + (P - b); }
inline u64 negm(u64 a) { return a ? P - a : 0; }
inline u64 mulm(u64 a, u64 b) { return (u64)(((u128)a * b) % P); }
inline u64 powm(u64 a, u128 e) {
    u64 r = 1;
    while (e) {
        if (e & 1) r = mulm(r, a);
        a = mulm(a, a);
        e >>= 1;
    }
    return r;
}
inline u64 invm(u64 a) { return powm(a, P - 2); }
inline u64 to_mont(u64 x) { return (u64)((((u128)x) << 64) % P); }                 // x * 2^64 mod p
inline u64 from_mont(u64 w) { return mulm(w, invm((u64)((((u128)1) << 64) % P))); }
constexpr u64 GENERATOR = 7;                                                        // Fp::GENERATOR
inline u64 two_adic_root() { return powm(GENERATOR, (P - 1) >> 32); }
inline u64 domain_generator(unsigned log_n) { return powm(two_adic_root(), (u128)1 << (32 - log_n)); }

struct Fq {   // Fq3 = Fp[X]/(X^3 - 2); an Fp element is (c0, 0, 0)
    u64 c[3] = {0, 0, 0};
    Fq() = default;
    Fq(u64 a) { c[0] = a % P; }
    Fq(u64 a, u64 b, u64 d) { c[0] = a; c[1] = b; c[2] = d; }
    bool operator==(const Fq &o) const { return c[0] == o.c[0] && c[1] == o.c[1] && c[2] == o.c[2]; }
    bool operator<(const Fq &o) const { return std::lexicographical_compare(c, c + 3, o.c, o.c + 3); }
    bool is_zero() const { return !(c[0] | c[1] | c[2]); }
};
inline Fq fq_add(const Fq &a, const Fq &b) { return Fq(addm(a.c[0], b.c[0]), addm(a.c[1], b.c[1]), addm(a.c[2], b.c[2])); }
inline Fq fq_neg(const Fq &a) { return Fq(negm(a.c[0]), negm(a.c[1]), negm(a.c[2])); }
inline Fq fq_sub(const Fq &a, const Fq &b) { return fq_add(a, fq_neg(b)); }
inline Fq fq_mul(const Fq &a, const Fq &b) {
    u64 pr[5] = {0, 0, 0, 0, 0};
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) pr[i + j] = addm(pr[i + j], mulm(a.c[i], b.c[j]));
    return Fq(addm(pr[0], mulm(2, pr[3])), addm(pr[1], mulm(2, pr[4])), pr[2]);
}
inline Fq fq_scale(const Fq &a, u64 s) { return Fq(mulm(a.c[0], s), mulm(a.c[1], s), mulm(a.c[2], s)); }
inline Fq fq_pow_big(Fq a, const std::vector<u64> &e_le) {   // exponent as little-endian 64-bit limbs
    Fq r(1);
    for (size_t l = 0; l < e_le.size(); l++)
        for (int b = 0; b < 64; b++) {
            if ((e_le[l] >> b) & 1) r = fq_mul(r, a);
            a = fq_mul(a, a);
        }
    return r;
}
inline Fq fq_pow(const Fq &a, u64 e) { return fq_pow_big(a, {e}); }
inline Fq fq_inv(const Fq &a) {
    // a^(p^3 - 2): p^3 - 2 as three 64-bit limbs
    u128 p2 = (u128)P * P;                                  // 128 bits
    u64 p2lo = (u64)p2, p2hi = (u64)(p2 >> 64);
    u128 lo = (u128)p2lo * P, hi = (u128)p2hi * P + (lo >> 64);
    std::vector<u64> e = {(u64)lo, (u64)hi, (u64)(hi >> 64)};
    // subtract 2
    if (e[0] >= 2) e[0] -= 2;
    else { e[0] -= 2; if (e[1]-- == 0) e[2]--; }
    return fq_pow_big(a, e);
}

// ------------------------------------------------------------------------------------------------ SHA-256 (host)
class Sha256 {
    u32 h[8];
    u8 buf[64];
    size_t fill = 0;
    u64 total = 0;
    static u32 rotr(u32 x, int r) { return (x >> r) | (x << (32 - r)); }
    void block(const u8 *p) {
        static const u32 K[64] = {
            0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
            0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
            0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
            0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
            0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
            0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
            0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};
        u32 w[64];
        for (int i = 0; i < 16; i++) w[i] = ((u32)p[4 * i] << 24) | ((u32)p[4 * i + 1] << 16) | ((u32)p[4 * i + 2] << 8) | p[4 * i + 3];
        for (int i = 16; i < 64; i++) {
            u32 s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3), s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
            w[i] = w[i - 16] + s0 + w[i - 7] + s1;
        }
        u32 a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
        for (int i = 0; i < 64; i++) {
            u32 t1 = hh + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + K[i] + w[i];
            u32 t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
            hh = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
        }
        h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e; h[5] += f; h[6] += g; h[7] += hh;
    }

public:
    Sha256() {
        static const u32 iv[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
        memcpy(h, iv, sizeof h);
    }
    Sha256 &update(const u8 *p, size_t n) {
        total += n;
        while (n) {
            size_t k = std::min(n, 64 - fill);
            memcpy(buf + fill, p, k);
            fill += k; p += k; n -= k;
            if (fill == 64) { block(buf); fill = 0; }
        }
        return *this;
    }
    Sha256 &update(const Bytes &b) { return update(b.data(), b.size()); }
    Bytes finish() {
        u64 bits = total * 8;
        u8 pad = 0x80;
        update(&pad, 1);
        u8 z = 0;
        while (fill != 56) update(&z, 1);
        u8 len[8];
        for (int i = 0; i < 8; i++) len[i] = (u8)(bits >> (56 - 8 * i));
        update(len, 8);
        Bytes out(32);
        for (int i = 0; i < 8; i++)
            for (int j = 0; j < 4; j++) out[4 * i + j] = (u8)(h[i] >> (24 - 8 * j));
        return out;
    }
};
inline Bytes sha256(std::initializer_list<Bytes> chunks) {
    Sha256 s;
    for (const Bytes &c : chunks) s.update(c);
    return s.finish();
}

// ------------------------------------------------------------------------------------------------ serialization
inline void put_u64_le(Bytes &o, u64 v) { for (int i = 0; i < 8; i++) o.push_back((u8)(v >> (8 * i))); }
inline Bytes be64(u64 v) { Bytes o(8); for (int i = 0; i < 8; i++) o[i] = (u8)(v >> (56 - 8 * i)); return o; }
// Field::serialize: 8-byte LE canonical integer per base-field limb
inline void put_elem(Bytes &o, const Fq &v, int lanes) { for (int l = 0; l < lanes; l++) put_u64_le(o, v.c[l]); }
inline void put_digest(Bytes &o, const Bytes &d) { put_u64_le(o, 32); o.insert(o.end(), d.begin(), d.end()); }

// ------------------------------------------------------------------------------------------------ public coin
class PublicCoin {   // PublicCoinImpl<F, Sha256HashFn>, src/random.rs:91-181
    u64 counter = 0;
    Bytes bytes;
    int lanes;       // 1: Field = Fp, 3: Field = Fq3
    void reset(Bytes s) { seed = std::move(s); counter = 0; bytes.clear(); }
    u8 next_byte() {
        if (bytes.empty()) { counter++; bytes = sha256({seed, be64(counter)}); }
        u8 b = bytes.back();                        // bytes are popped from the END of hash(seed || counter)
        bytes.pop_back();
        return b;
    }
    u64 draw_fp() {
        for (;;) {                                  // raw u64 below p taken as the Montgomery word (SURVEY.md 8c)
            u64 w = next_u64();
            if (w < P) return from_mont(w);
        }
    }

public:
    Bytes seed;
    PublicCoin(Bytes s, int field_lanes) : lanes(field_lanes), seed(std::move(s)) {}
    void reseed_with_digest(const Bytes &d) { reset(sha256({seed, d})); }
    void reseed_with_field_elements(const std::vector<Fq> &vals) {
        for (const Fq &v : vals) {
            Bytes ser;
            put_elem(ser, v, lanes);
            reset(sha256({seed, sha256({ser})}));
        }
    }
    void reseed_with_int(u64 v) { reset(sha256({seed, be64(v)})); }
    static unsigned leading_zeros(const Bytes &d) {
        unsigned z = 0;
        for (u8 b : d) {
            if (b == 0) { z += 8; continue; }
            z += (unsigned)__builtin_clz((unsigned)b) - 24;
            break;
        }
        return z;
    }
    bool verify_proof_of_work(unsigned bits, u64 nonce) const { return leading_zeros(sha256({seed, be64(nonce)})) >= bits; }
    u64 next_u64() {
        u64 v = 0;
        for (int i = 0; i < 8; i++) v = (v << 8) | next_byte();
        return v;
    }
    Fq draw() {
        if (lanes != 3) return Fq(draw_fp());
        const u64 c0 = draw_fp(), c1 = draw_fp(), c2 = draw_fp();     // c0, c1, c2 in this order (argument evaluation order is unspecified)
        return Fq(c0, c1, c2);
    }
    std::vector<u64> draw_queries(unsigned max_n, u64 domain_size) {   // rand 0.8.5 gen_range: widening multiply + zone
        const u64 zone = (domain_size << __builtin_clzll(domain_size)) - 1;
        std::set<u64> out;
        for (unsigned i = 0; i < max_n; i++)
            for (;;) {
                u128 m = (u128)next_u64() * domain_size;
                if ((u64)m <= zone) { out.insert((u64)(m >> 64)); break; }
            }
        return std::vector<u64>(out.begin(), out.end());
    }
};

// ------------------------------------------------------------------------------------------------ proof objects
struct ProofOptions {
    u8 num_queries, lde_blowup_factor, grinding_factor, fri_folding_factor, fri_max_remainder_coeffs;
    Bytes to_bytes() const { return {num_queries, lde_blowup_factor, grinding_factor, fri_folding_factor, fri_max_remainder_coeffs}; }
    unsigned fri_num_layers(u64 domain) const {
        unsigned k = 0;
        while (domain > (u64)fri_max_remainder_coeffs * lde_blowup_factor) { domain /= fri_folding_factor; k++; }
        return k;
    }
    bool operator<(const ProofOptions &o) const { return to_bytes() < o.to_bytes(); }
};
struct MerkleView {
    std::vector<Bytes> nodes, initial_leaves, sibling_leaves;
    u32 height = 0;
    void write(Bytes &o) const {
        for (const auto *v : {&nodes, &initial_leaves, &sibling_leaves}) {
            put_u64_le(o, v->size());
            for (const Bytes &d : *v) put_digest(o, d);
        }
        for (int i = 0; i < 4; i++) o.push_back((u8)(height >> (8 * i)));
    }
};
struct LayerProof {
    std::vector<Fq> flattenend_rows;
    MerkleView merkle_proof;
    Bytes commitment;
};
struct FriProof {
    std::vector<LayerProof> layers;
    std::vector<Fq> remainder_coeffs;
};
struct Queries {
    std::vector<Fq> base_trace_values, extension_trace_values, composition_trace_values;
    MerkleView base_trace_proof, composition_trace_proof;
    bool has_extension = false;
    MerkleView extension_trace_proof;
};
struct Proof {
    ProofOptions options;
    u64 trace_len = 0;
    Bytes base_trace_commitment, composition_trace_commitment;
    bool has_extension = false;
    Bytes extension_trace_commitment;
    FriProof fri_proof;
    u64 pow_nonce = 0;
    Queries trace_queries;
    std::vector<Fq> execution_trace_ood_evals, composition_trace_ood_evals;

    // ark-serialize layout (compressed): fields in declaration order, Vec = u64 length + items, Option = tag byte
    Bytes to_bytes(int fq_lanes) const {
        Bytes o = options.to_bytes();
        auto vec = [&](const std::vector<Fq> &v, int lanes) { put_u64_le(o, v.size()); for (const Fq &e : v) put_elem(o, e, lanes); };
        put_u64_le(o, trace_len);
        put_digest(o, base_trace_commitment);
        o.push_back(has_extension ? 1 : 0);
        if (has_extension) put_digest(o, extension_trace_commitment);
        put_digest(o, composition_trace_commitment);
        put_u64_le(o, fri_proof.layers.size());
        for (const LayerProof &l : fri_proof.layers) {
            vec(l.flattenend_rows, fq_lanes);
            l.merkle_proof.write(o);
            put_digest(o, l.commitment);
        }
        vec(fri_proof.remainder_coeffs, fq_lanes);
        put_u64_le(o, pow_nonce);
        vec(trace_queries.base_trace_values, 1);
        vec(trace_queries.extension_trace_values, fq_lanes);
        vec(trace_queries.composition_trace_values, fq_lanes);
        trace_queries.base_trace_proof.write(o);
        o.push_back(trace_queries.has_extension ? 1 : 0);
        if (trace_queries.has_extension) trace_queries.extension_trace_proof.write(o);
        trace_queries.composition_trace_proof.write(o);
        vec(execution_trace_ood_evals, fq_lanes);
        vec(composition_trace_ood_evals, fq_lanes);
        return o;
    }
};

// ------------------------------------------------------------------------------------------------ expressions
// Hash-consed DAG in an arena; an Expr is (graph, node id).  Leaves: X | Const | Challenge | Hint | CompositionCoeff |
// Trace(column, offset); nodes: Neg | Add | Mul | Div | Pow(usize) (src/expression.rs:31-39); Inv appears only inside the
// compiler (a / b is evaluated as a * inv(b) with inv(b) shared).
enum Kind : int { K_X, K_CONST, K_CHAL, K_HINT, K_CCOEF, K_TRACE, K_NEG, K_ADD, K_MUL, K_DIV, K_POW, K_INV };
struct Node {
    Kind kind;
    int a = -1, b = -1;      // children
    u64 k[3] = {0, 0, 0};    // constant value | index | (column, offset as two's complement) | exponent
    bool ext = false;        // constants: extension-typed
};
class Graph {
    std::map<std::tuple<int, int, int, u64, u64, u64, bool>, int> pool;

public:
    std::vector<Node> nodes;
    int mk(Kind kind, int a = -1, int b = -1, u64 k0 = 0, u64 k1 = 0, u64 k2 = 0, bool ext = false) {
        auto key = std::make_tuple((int)kind, a, b, k0, k1, k2, ext);
        auto it = pool.find(key);
        if (it != pool.end()) return it->second;
        Node n;
        n.kind = kind; n.a = a; n.b = b; n.k[0] = k0; n.k[1] = k1; n.k[2] = k2; n.ext = ext;
        nodes.push_back(n);
        return pool[key] = (int)nodes.size() - 1;
    }
};
struct Expr {
    Graph *g = nullptr;
    int id = -1;
    Expr operator+(const Expr &o) const { return {g, g->mk(K_ADD, id, o.id)}; }
    Expr operator-() const { return {g, g->mk(K_NEG, id)}; }
    Expr operator-(const Expr &o) const { return *this + (-o); }     // a - b = a + (-b), as the reference's Sub
    Expr operator*(const Expr &o) const { return {g, g->mk(K_MUL, id, o.id)}; }
    Expr operator/(const Expr &o) const { return {g, g->mk(K_DIV, id, o.id)}; }
    Expr pow(u64 e) const { return {g, g->mk(K_POW, id, -1, e)}; }
};
inline Expr X(Graph &g) { return {&g, g.mk(K_X)}; }
inline Expr Constant(Graph &g, u64 v) { return {&g, g.mk(K_CONST, -1, -1, v % P, 0, 0, false)}; }
inline Expr ConstantQ(Graph &g, const Fq &v) { return {&g, g.mk(K_CONST, -1, -1, v.c[0], v.c[1], v.c[2], true)}; }
inline Expr Challenge(Graph &g, u64 i) { return {&g, g.mk(K_CHAL, -1, -1, i)}; }
inline Expr Hint(Graph &g, u64 i) { return {&g, g.mk(K_HINT, -1, -1, i)}; }
inline Expr CompositionCoeff(Graph &g, u64 i) { return {&g, g.mk(K_CCOEF, -1, -1, i)}; }
inline Expr Trace(Graph &g, u64 col, int64_t off) { return {&g, g.mk(K_TRACE, -1, -1, col, (u64)off)}; }

// post-order of the sub-DAG under `root` (children before parents), optional child ordering by sub-DAG size
inline std::vector<int> post_order(const Graph &g, int root, bool big_first) {
    std::vector<u64> size(g.nodes.size(), 0);
    std::vector<char> seen(g.nodes.size(), 0);
    std::vector<int> order;
    if (big_first) {   // node ids are topological (children are created before parents): one forward sweep
        for (size_t i = 0; i < g.nodes.size(); i++) size[i] = 1 + (g.nodes[i].a >= 0 ? size[g.nodes[i].a] : 0) + (g.nodes[i].b >= 0 ? size[g.nodes[i].b] : 0);
    }
    std::vector<std::pair<int, bool>> st = {{root, false}};
    while (!st.empty()) {
        auto [n, done] = st.back();
        st.pop_back();
        if (done) { order.push_back(n); continue; }
        if (seen[n]) continue;
        seen[n] = 1;
        st.push_back({n, true});
        int kids[2], nk = 0;
        if (g.nodes[n].a >= 0 && !seen[g.nodes[n].a]) kids[nk++] = g.nodes[n].a;
        if (g.nodes[n].b >= 0 && g.nodes[n].b != g.nodes[n].a && !seen[g.nodes[n].b]) kids[nk++] = g.nodes[n].b;
        if (nk == 2 && big_first && size[kids[0]] > size[kids[1]]) std::swap(kids[0], kids[1]);   // popped LIFO: largest first
        for (int i = 0; i < nk; i++) st.push_back({kids[i], false});
    }
    return order;
}

// (numerator degree, denominator degree) by the reference's rules (src/constraints.rs:404-455)
inline std::pair<u64, u64> degree(const Graph &g, int root, u64 trace_degree) {
    std::vector<std::pair<u64, u64>> d(g.nodes.size());
    for (int n : post_order(g, root, false)) {
        const Node &nd = g.nodes[n];
        switch (nd.kind) {
            case K_CONST: case K_CHAL: case K_HINT: case K_CCOEF: d[n] = {0, 0}; break;
            case K_TRACE: d[n] = {trace_degree, 0}; break;
            case K_X: d[n] = {1, 0}; break;
            case K_NEG: d[n] = d[nd.a]; break;
            case K_ADD: d[n] = {std::max(d[nd.a].first + d[nd.b].second, d[nd.b].first + d[nd.a].second), d[nd.a].second + d[nd.b].second}; break;
            case K_MUL: d[n] = {d[nd.a].first + d[nd.b].first, d[nd.a].second + d[nd.b].second}; break;
            case K_DIV: d[n] = {d[nd.a].first + d[nd.b].second, d[nd.a].second + d[nd.b].first}; break;
            case K_POW: d[n] = {d[nd.a].first * nd.k[0], d[nd.a].second * nd.k[0]}; break;
            default: throw std::runtime_error("degree: unsupported node");
        }
    }
    return d[root];
}
inline u64 ceil_power_of_two(u64 v) {
    if (v == 0) return 1;
    if ((v & (v - 1)) == 0) return v;
    return (u64)1 << (64 - __builtin_clzll(v));
}
inline u64 blowup_factor(const Graph &g, int root, u64 trace_len) {
    auto [num, den] = degree(g, root, trace_len - 1);
    return ceil_power_of_two(num > den ? num - den : 0) / (trace_len - 1);
}

// ------------------------------------------------------------------------------------------------ evaluator programs
enum Op : u32 { OP_X = 0, OP_CONST, OP_TRACE, OP_NEG, OP_ADD, OP_SUB, OP_MUL, OP_INV, OP_POW, OP_STORE, OP_PERIODIC };   // csrc/eval.cu (OP_PERIODIC: periodic columns, emitted by the Python compiler only)
constexpr int MAX_REGS = 48;
struct Binding { u32 slot; Kind kind; u64 index; };
struct Program {
    std::vector<std::array<u32, 4>> code;
    std::vector<std::array<u64, 3>> consts;     // Montgomery words
    std::vector<Binding> bindings;
    int nregs = 0;
    // fill the symbolic constants with this proof's randomness (canonical values)
    Program bind(const std::vector<Fq> &challenges, const std::vector<Fq> &hints, const std::vector<Fq> &ccoefs) const {
        Program p = *this;
        for (const Binding &b : bindings) {
            const std::vector<Fq> &src = b.kind == K_CHAL ? challenges : (b.kind == K_HINT ? hints : ccoefs);
            const Fq &v = src.at(b.index);
            p.consts[b.slot] = {to_mont(v.c[0]), to_mont(v.c[1]), to_mont(v.c[2])};
        }
        return p;
    }
};

// Flatten the DAG under `root` into the evaluator's linear program (the algorithm of ministark_b200/expr.py::compile_program
// with symbolic = true): a / b -> a * inv(b) with shared inverses; constant folding; largest-operand-first post order;
// registers by liveness with least-recently-used eviction of rematerialisable leaves (x, trace loads, constants).
// Montgomery's trick inside one evaluation point (ministark_b200/expr.py::_batch_inverses): the inverses 1/d_1 .. 1/d_k whose
// operands are functions of the point alone (x, constants; no trace cell, no inverse inside) become ONE inversion of
// d_1 ... d_k and 3(k - 1) multiplications, per field.  For programs whose denominators cannot vanish on the evaluation
// domain (the AIR composition and the DEEP polynomial over the LDE coset): with a zero operand every inverse of the batch
// would come out 0, where independent inversions only zero their own term (src/eval_cpu.rs:280-295).
inline int batch_inverses_pass(Graph &g, int root, u32 num_base_cols) {
    const std::vector<int> post = post_order(g, root, false);
    std::map<int, char> has_inv, varies, reads_trace, typ;
    for (int n : post) {
        const Node &nd = g.nodes[n];
        const bool ka = nd.a >= 0, kb = nd.b >= 0;
        has_inv[n] = nd.kind == K_INV || (ka && has_inv[nd.a]) || (kb && has_inv[nd.b]);
        varies[n] = nd.kind == K_X || nd.kind == K_TRACE || (ka && varies[nd.a]) || (kb && varies[nd.b]);
        reads_trace[n] = nd.kind == K_TRACE || (ka && reads_trace[nd.a]) || (kb && reads_trace[nd.b]);
        switch (nd.kind) {
            case K_CONST: typ[n] = nd.ext; break;
            case K_CHAL: case K_HINT: case K_CCOEF: typ[n] = 1; break;
            case K_X: typ[n] = 0; break;
            case K_TRACE: typ[n] = nd.k[0] >= num_base_cols; break;
            default: typ[n] = std::max(ka ? typ[nd.a] : (char)0, kb ? typ[nd.b] : (char)0);
        }
    }
    std::map<int, int> repl;
    for (char field = 0; field < 2; field++) {
        std::vector<int> members;
        for (int n : post)
            if (g.nodes[n].kind == K_INV && typ[n] == field && varies[g.nodes[n].a] && !has_inv[g.nodes[n].a] && !reads_trace[g.nodes[n].a])
                members.push_back(n);
        if (members.size() < 2) continue;
        std::vector<int> ds, prefix;
        for (int m : members) ds.push_back(g.nodes[m].a);
        prefix.push_back(ds[0]);
        for (size_t i = 1; i < ds.size(); i++) prefix.push_back(g.mk(K_MUL, prefix.back(), ds[i]));
        int inv = g.mk(K_INV, prefix.back());
        for (size_t i = ds.size() - 1; i >= 1; i--) {
            repl[members[i]] = g.mk(K_MUL, inv, prefix[i - 1]);
            inv = g.mk(K_MUL, inv, ds[i]);
        }
        repl[members[0]] = inv;
    }
    if (repl.empty()) return root;
    std::map<int, int> rebuilt;
    for (int n : post) {
        if (repl.count(n)) { rebuilt[n] = repl[n]; continue; }
        const Node nd = g.nodes[n];
        rebuilt[n] = g.mk(nd.kind, nd.a >= 0 ? rebuilt[nd.a] : -1, nd.b >= 0 ? rebuilt[nd.b] : -1, nd.k[0], nd.k[1], nd.k[2], nd.ext);
    }
    return rebuilt[root];
}

inline Program compile_program(Graph &g, int root, u32 num_base_cols, u64 lde_step, int log_ce, bool batch_inverses = false) {
    // ---- rewrite Div; split the degree-adjustment powers x^(a n + b) into (x^n)^a * x^b, which share the squarings of x^n
    const u64 trace_len = (log_ce >= 0 && lde_step >= 1) ? (((u64)1 << log_ce) / lde_step) : 0;
    std::vector<int> rew(g.nodes.size(), -1);
    for (int n : post_order(g, root, false)) {
        const Node nd = g.nodes[n];
        const int a = nd.a >= 0 ? rew[nd.a] : -1, b = nd.b >= 0 ? rew[nd.b] : -1;
        if (nd.kind == K_DIV) {
            rew[n] = g.mk(K_MUL, a, g.mk(K_INV, b));
        } else if (nd.kind == K_POW && g.nodes[a].kind == K_X && trace_len && nd.k[0] >= 2 * trace_len && nd.k[0] % trace_len < 64) {
            const u64 a_ = nd.k[0] / trace_len, b_ = nd.k[0] % trace_len;
            int v = g.mk(K_POW, a, -1, trace_len);
            if (a_ > 1) v = g.mk(K_POW, v, -1, a_);
            if (b_) v = g.mk(K_MUL, v, b_ > 1 ? g.mk(K_POW, a, -1, b_) : a);
            rew[n] = v;
        } else {
            rew[n] = g.mk(nd.kind, a, b, nd.k[0], nd.k[1], nd.k[2], nd.ext);
        }
        if (rew.size() < g.nodes.size()) rew.resize(g.nodes.size(), -1);
    }
    root = rew[root];
    if (batch_inverses) root = batch_inverses_pass(g, root, num_base_cols);
    const std::vector<int> order = post_order(g, root, true);
    // ---- constant folding + typing (0 = Fp, 1 = Fq)
    const size_t NN = g.nodes.size();
    std::vector<char> has_c(NN, 0), typ(NN, 0);
    std::vector<Fq> cval(NN);
    auto symbolic = [&](int n) { Kind k = g.nodes[n].kind; return k == K_CHAL || k == K_HINT || k == K_CCOEF; };
    for (int n : order) {
        const Node &nd = g.nodes[n];
        switch (nd.kind) {
            case K_CONST: has_c[n] = 1; cval[n] = Fq(nd.k[0], nd.k[1], nd.k[2]); typ[n] = nd.ext; break;
            case K_CHAL: case K_HINT: case K_CCOEF: typ[n] = 1; break;
            case K_X: typ[n] = 0; break;
            case K_TRACE: typ[n] = nd.k[0] >= num_base_cols; break;
            default: {
                typ[n] = std::max(typ[nd.a], nd.b >= 0 ? typ[nd.b] : (char)0);
                const bool all = has_c[nd.a] && (nd.b < 0 || has_c[nd.b]);
                if (all) {
                    has_c[n] = 1;
                    switch (nd.kind) {
                        case K_NEG: cval[n] = fq_neg(cval[nd.a]); break;
                        case K_ADD: cval[n] = fq_add(cval[nd.a], cval[nd.b]); break;
                        case K_MUL: cval[n] = fq_mul(cval[nd.a], cval[nd.b]); break;
                        case K_INV: cval[n] = fq_inv(cval[nd.a]); break;
                        case K_POW: cval[n] = fq_pow(cval[nd.a], nd.k[0]); break;
                        default: throw std::runtime_error("fold: unsupported node");
                    }
                }
            }
        }
    }
    // ---- live nodes and last uses
    std::vector<int> live;
    for (int n : order)
        if (!has_c[n] || n == root) live.push_back(n);
    std::vector<int> last_use(NN, -1);
    for (size_t idx = 0; idx < live.size(); idx++) {
        const Node &nd = g.nodes[live[idx]];
        if (nd.a >= 0) last_use[nd.a] = (int)idx;
        if (nd.b >= 0) last_use[nd.b] = (int)idx;
    }
    Program P;
    std::map<Fq, u32> const_idx;
    auto const_slot = [&](const Fq &v) {
        auto it = const_idx.find(v);
        if (it != const_idx.end()) return it->second;
        P.consts.push_back({to_mont(v.c[0]), to_mont(v.c[1]), to_mont(v.c[2])});
        return const_idx[v] = (u32)P.consts.size() - 1;
    };
    std::map<std::pair<int, u64>, u32> sym_slot;
    std::vector<int> reg_of(NN, -1), free_regs;
    std::set<int> leaf_regs, pinned;
    std::vector<long> touch(NN, -1);
    int nregs = 0;
    auto is_leaf = [&](int n) { Kind k = g.nodes[n].kind; return has_c[n] || k == K_X || k == K_TRACE || symbolic(n); };
    auto alloc = [&]() {
        if (!free_regs.empty()) { int r = free_regs.back(); free_regs.pop_back(); return r; }
        if (nregs < MAX_REGS) return nregs++;
        int victim = -1;
        for (int n : leaf_regs)
            if (!pinned.count(n) && (victim < 0 || touch[n] < touch[victim])) victim = n;
        if (victim < 0) throw std::runtime_error("expression needs more than 48 live temporaries");
        leaf_regs.erase(victim);
        int r = reg_of[victim];
        reg_of[victim] = -1;
        return r;
    };
    auto emit_leaf = [&](int n) {
        const int r = alloc();
        const Node &nd = g.nodes[n];
        if (has_c[n]) {
            P.code.push_back({(u32)OP_CONST | ((u32)typ[n] << 8), (u32)r, const_slot(cval[n]), 0});
        } else if (symbolic(n)) {
            auto key = std::make_pair((int)nd.kind, nd.k[0]);
            if (!sym_slot.count(key)) {
                sym_slot[key] = (u32)P.consts.size();
                P.consts.push_back({0, 0, 0});
                P.bindings.push_back({sym_slot[key], nd.kind, nd.k[0]});
            }
            P.code.push_back({(u32)OP_CONST | (1u << 8), (u32)r, sym_slot[key], 0});
        } else if (nd.kind == K_X) {
            P.code.push_back({(u32)OP_X, (u32)r, 0, 0});
        } else {
            int64_t shift = (int64_t)lde_step * (int64_t)nd.k[1];
            if (log_ce >= 0) shift = ((shift % ((int64_t)1 << log_ce)) + ((int64_t)1 << log_ce)) % ((int64_t)1 << log_ce);
            P.code.push_back({(u32)OP_TRACE | ((u32)(nd.k[0] >= num_base_cols) << 8), (u32)r, (u32)nd.k[0], (u32)shift});
        }
        reg_of[n] = r;
        leaf_regs.insert(n);
        return r;
    };
    auto operand = [&](int n) {
        const int r = reg_of[n] >= 0 ? reg_of[n] : emit_leaf(n);
        pinned.insert(n);
        touch[n] = (long)P.code.size();
        return r;
    };
    auto release = [&](int n, int idx) {
        if (last_use[n] == idx && reg_of[n] >= 0) {
            free_regs.push_back(reg_of[n]);
            reg_of[n] = -1;
            leaf_regs.erase(n);
        }
    };
    for (size_t idx = 0; idx < live.size(); idx++) {
        const int n = live[idx];
        const Node &nd = g.nodes[n];
        pinned.clear();
        if (is_leaf(n)) {
            if (n == root) operand(n);
            continue;
        }
        int r;
        if (nd.kind == K_ADD || nd.kind == K_MUL) {
            const int ra = operand(nd.a), rb = operand(nd.b);
            release(nd.a, (int)idx);
            release(nd.b, (int)idx);
            r = alloc();
            P.code.push_back({(u32)(nd.kind == K_ADD ? OP_ADD : OP_MUL) | ((u32)typ[nd.a] << 8) | ((u32)typ[nd.b] << 9), (u32)r, (u32)ra, (u32)rb});
        } else if (nd.kind == K_NEG || nd.kind == K_INV || nd.kind == K_POW) {
            const int ra = operand(nd.a);
            release(nd.a, (int)idx);
            r = alloc();
            const u32 op = nd.kind == K_NEG ? OP_NEG : (nd.kind == K_INV ? OP_INV : OP_POW);
            if (nd.kind == K_POW && nd.k[0] >= ((u64)1 << 32)) throw std::runtime_error("exponent too large");
            P.code.push_back({op | ((u32)typ[nd.a] << 8), (u32)r, (u32)ra, nd.kind == K_POW ? (u32)nd.k[0] : 0u});
        } else {
            throw std::runtime_error("compile: unsupported node");
        }
        reg_of[n] = r;
    }
    P.code.push_back({(u32)OP_STORE | ((u32)typ[root] << 8), 0, (u32)reg_of[root], 0});
    P.nregs = std::max(nregs, 1);
    return P;
}

// ------------------------------------------------------------------------------------------------ AIR bookkeeping
struct AirConfig {
    u32 num_base_columns = 0, num_extension_columns = 0;
    bool fq_is_fp = true;
    std::function<std::vector<Expr>(Graph &, u64 trace_len)> constraints;
    std::function<std::vector<Fq>(u64 trace_len, const std::vector<Fq> &public_inputs, const std::vector<Fq> &challenges)> gen_hints;
};
class Air {   // Air::new (src/air.rs:142-160) + AirConfig::composition_constraint (src/air.rs:50-82)
public:
    Graph g;
    u64 trace_len;
    unsigned log_n;
    ProofOptions options;
    std::vector<Expr> constraints;
    Expr composition;
    u64 ce_blowup_factor = 1;
    Air(const AirConfig &cfg, u64 n, ProofOptions opts) : trace_len(n), options(opts) {
        log_n = 63 - (unsigned)__builtin_clzll(n);
        constraints = cfg.constraints(g, n);
        u64 ce = 0;
        for (const Expr &c : constraints) ce = std::max(ce, blowup_factor(g, c.id, n));
        const u64 composition_degree = n * ce - 1;
        Expr x = X(g), total;
        for (size_t i = 0; i < constraints.size(); i++) {
            auto [num, den] = degree(g, constraints[i].id, n - 1);
            if (num - den > composition_degree) throw std::runtime_error("constraint degree exceeds the composition degree");
            const u64 adj = composition_degree - (num - den);
            Expr term = constraints[i] * (x.pow(adj) * CompositionCoeff(g, 2 * i) + CompositionCoeff(g, 2 * i + 1));
            total = i == 0 ? term : total + term;
        }
        composition = total;
        ce_blowup_factor = blowup_factor(g, composition.id, n);
        if (ce_blowup_factor > opts.lde_blowup_factor) throw std::runtime_error("ce blow-up exceeds the LDE blow-up");
    }
    u64 max_leaf_index(Kind kind) const {   // number of challenges / composition coefficients = max index + 1
        u64 m = 0;
        bool any = false;
        for (const Node &nd : g.nodes)
            if (nd.kind == kind) { m = std::max(m, nd.k[0]); any = true; }
        return any ? m + 1 : 0;
    }
    u64 num_challenges() const { return max_leaf_index(K_CHAL); }
    u64 num_composition_constraint_coeffs() const { return max_leaf_index(K_CCOEF); }
    std::vector<std::pair<u64, int64_t>> trace_arguments() const {   // BTreeSet<(column, offset)>: sorted
        std::set<std::pair<u64, int64_t>> s;
        for (const Expr &c : constraints)
            for (int n : post_order(g, c.id, false))
                if (g.nodes[n].kind == K_TRACE) s.insert({g.nodes[n].k[0], (int64_t)g.nodes[n].k[1]});
        return std::vector<std::pair<u64, int64_t>>(s.begin(), s.end());
    }
    Program composition_program(u32 num_base_cols) {
        int log_ce = (int)log_n + (63 - __builtin_clzll(ce_blowup_factor));
        return compile_program(g, composition.id, num_base_cols, ce_blowup_factor, log_ce, /*batch_inverses=*/true);   // zerofier denominators
    }
    // the same constraints over one coset block of n rows (ministark_b200/cosets.py::block_program): inside a block the
    // ce-domain stride is 1 and the domain has n points
    Program block_program(u32 num_base_cols) {
        return compile_program(g, composition.id, num_base_cols, 1, (int)log_n, /*batch_inverses=*/true);
    }
};

// examples/fib (examples/fib/main.rs:78-150): 8 boundary + 1 terminal + 8 transition constraints
inline AirConfig fib_air_config() {
    AirConfig cfg;
    cfg.num_base_columns = 8;
    cfg.fq_is_fp = true;
    cfg.gen_hints = [](u64, const std::vector<Fq> &pub, const std::vector<Fq> &) { return std::vector<Fq>{pub.at(0)}; };
    cfg.constraints = [](Graph &g, u64 n) {
        const unsigned log_n = 63 - (unsigned)__builtin_clzll(n);
        Expr x = X(g), one = Constant(g, 1), first = Constant(g, 1), last = Constant(g, powm(domain_generator(log_n), n - 1));
        std::vector<Expr> v = {one, one + one};
        v.push_back(v[1] * v[0]);
        for (int i = 3; i < 8; i++) v.push_back(v[i - 2] * v[i - 1]);
        auto T = [&](u64 c, int64_t o) { return Trace(g, c, o); };
        std::vector<Expr> out;
        for (int i = 0; i < 8; i++) out.push_back((T(i, 0) - v[i]) / (x - first));
        out.push_back((T(7, 0) - Hint(g, 0)) / (x - last));
        Expr but_last = (x - last) / (x.pow(n) - one);
        out.push_back((T(0, 1) - T(6, 0) * T(7, 0)) * but_last);
        out.push_back((T(1, 1) - T(7, 0) * T(0, 1)) * but_last);
        for (int k = 2; k < 8; k++) out.push_back((T(k, 1) - T(k - 2, 1) * T(k - 1, 1)) * but_last);
        return out;
    };
    return cfg;
}

}  // namespace mshost
