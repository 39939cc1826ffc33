// plonky2_b200.hpp -- C++17 host layer over the C ABI (plonky2_b200.h), mirroring the reference's Rust
// interface for the prover hot path: same type and function names, argument meaning and error behaviour, so
// that host code (and tests) read like the reference's own. Header-only; needs only libplonky2_b200.so.
//
//   reference (Rust)                                         here (namespace plonky2_b200)
//   field/src/fft.rs:53-91            fft_with_options ...   fft_with_options / ifft_with_options / coset_fft
//   plonky2/src/hash/hash_types.rs    HashOut                HashOut
//   plonky2/src/hash/merkle_tree.rs   MerkleCap, MerkleProof MerkleCap, MerkleProof
//   plonky2/src/iop/challenger.rs     Challenger             Challenger (host, sequential, as in the reference)
//   plonky2/src/fri/oracle.rs         PolynomialBatch        PolynomialBatch (device-resident behind a handle)
//   plonky2/src/fri/mod.rs            FriConfig, FriParams   FriConfig, FriParams
//   plonky2/src/fri/reduction_strategies.rs                  FriReductionStrategy
//   plonky2/src/fri/structure.rs      FriInstanceInfo ...    FriInstanceInfo, FriBatchInfo, FriPolynomialInfo
//   plonky2/src/fri/proof.rs          FriProof ...           FriProof (+ to_bytes = write_fri_proof)
//   plonky2/src/fri/oracle.rs:176     prove_openings         PolynomialBatch::prove_openings
//
// Shape violations that panic in the reference throw ShapeError; other failures throw Error. There is no CPU
// fallback: constructing a Context without a CUDA device throws.
#pragma once
#include <array>
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "plonky2_b200.h"

namespace plonky2_b200 {

using F = uint64_t;                       // GoldilocksField(pub u64), field/src/goldilocks_field.rs:23-25
constexpr F ORDER = 0xFFFFFFFF00000001ULL;
constexpr int D = 2;                      // PoseidonGoldilocksConfig extension degree
struct Ext {                              // F::Extension = QuadraticExtension<F>, X^2 = 7
    F c0 = 0, c1 = 0;
};
constexpr size_t SALT_SIZE = GL_SALT_SIZE;
constexpr size_t SPONGE_RATE = 8, SPONGE_WIDTH = 12, NUM_HASH_OUT_ELTS = 4;

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
struct ShapeError : Error {
    using Error::Error;
};
inline void check(int rc, const gl_ctx* ctx = nullptr) {
    if (rc == GL_OK) return;
    const char* m = gl_last_error(ctx);
    std::string msg = m ? m : "plonky2_b200 error";
    if (rc == GL_ERR_BAD_SHAPE) throw ShapeError(rc, msg);
    throw Error(rc, msg);
}
inline uint32_t log2_strict(size_t n) {
    uint32_t l = 0;
    while ((size_t(1) << l) < n) l++;
    if ((size_t(1) << l) != n || n == 0) throw ShapeError(GL_ERR_BAD_SHAPE, "Not a power of two: " + std::to_string(n));
    return l;
}
// host scalar helpers (python-int free): a*b mod p via __int128
inline F fmul(F a, F b) { return (F)(((unsigned __int128)(a % ORDER) * (b % ORDER)) % ORDER); }
inline F fpow(F a, uint64_t e) {
    F r = 1;
    for (; e; e >>= 1, a = fmul(a, a))
        if (e & 1) r = fmul(r, a);
    return r;
}
inline F primitive_root_of_unity(uint32_t n_log) { return fpow(7277203076849721926ULL, uint64_t(1) << (32 - n_log)); }
inline Ext ext_mul(Ext a, Ext b) {
    auto add = [](F x, F y) { return (F)(((unsigned __int128)x + y) % ORDER); };
    return Ext{add(fmul(a.c0, b.c0), fmul(7, fmul(a.c1, b.c1))), add(fmul(a.c0, b.c1), fmul(a.c1, b.c0))};
}

class Context {
   public:
    explicit Context(int device = 0, void* stream = nullptr) { check(gl_ctx_create(device, stream, &h_)); }
    ~Context() { gl_ctx_destroy(h_); }
    Context(const Context&) = delete;
    Context& operator=(const Context&) = delete;
    gl_ctx* get() const { return h_; }
    uint64_t launch_count() const { return gl_ctx_launch_count(h_); }

   private:
    gl_ctx* h_ = nullptr;
};

// ---- NTT (field/src/fft.rs:53-91, polynomial/mod.rs:63-73,280-293) ----
inline std::vector<F> fft_with_options(Context& ctx, std::vector<F> coeffs, uint32_t zero_factor = 0) {
    check(gl_ntt(ctx.get(), coeffs.data(), log2_strict(coeffs.size()), 1, coeffs.size(), 0, zero_factor, 1, GL_MEM_HOST), ctx.get());
    return coeffs;
}
inline std::vector<F> ifft_with_options(Context& ctx, std::vector<F> values) {
    check(gl_ntt(ctx.get(), values.data(), log2_strict(values.size()), 1, values.size(), 1, 0, 1, GL_MEM_HOST), ctx.get());
    return values;
}
inline std::vector<F> coset_fft(Context& ctx, std::vector<F> coeffs, F shift) {
    check(gl_ntt(ctx.get(), coeffs.data(), log2_strict(coeffs.size()), 1, coeffs.size(), 0, 0, shift, GL_MEM_HOST), ctx.get());
    return coeffs;
}

// ---- hashes ----
struct HashOut {
    F elements[4] = {0, 0, 0, 0};
    bool operator==(const HashOut& o) const { return std::memcmp(elements, o.elements, 32) == 0; }
};
struct MerkleCap {
    std::vector<HashOut> hashes;
    size_t len() const { return hashes.size(); }
    size_t height() const { return log2_strict(hashes.size()); }
    std::vector<F> flatten() const {
        std::vector<F> v;
        for (auto& h : hashes) v.insert(v.end(), h.elements, h.elements + 4);
        return v;
    }
};
struct MerkleProof {
    std::vector<HashOut> siblings;
};

// ---- Challenger (iop/challenger.rs:16-153); the permutation is gl_poseidon_permute_host ----
class Challenger {
   public:
    Challenger() { std::memset(sponge_state_, 0, sizeof(sponge_state_)); }
    void observe_element(F e) {
        output_buffer_.clear();
        input_buffer_.push_back(e % ORDER);
        if (input_buffer_.size() == SPONGE_RATE) duplexing();
    }
    void observe_elements(const std::vector<F>& es) {
        for (F e : es) observe_element(e);
    }
    void observe_extension_element(Ext e) {
        observe_element(e.c0);
        observe_element(e.c1);
    }
    void observe_hash(const HashOut& h) {
        for (F e : h.elements) observe_element(e);
    }
    void observe_cap(const MerkleCap& cap) {
        for (auto& h : cap.hashes) observe_hash(h);
    }
    F get_challenge() {
        if (!input_buffer_.empty() || output_buffer_.empty()) duplexing();
        F v = output_buffer_.back();
        output_buffer_.pop_back();
        return v;
    }
    std::vector<F> get_n_challenges(size_t n) {
        std::vector<F> v(n);
        for (auto& x : v) x = get_challenge();
        return v;
    }
    Ext get_extension_challenge() {
        F a = get_challenge(), b = get_challenge();
        return Ext{a, b};
    }
    // for fri_proof_of_work (prover.rs:171-181): state with the pending inputs written in, and their count
    size_t duplex_intermediate_state(F out[12]) const {
        std::memcpy(out, sponge_state_, sizeof(sponge_state_));
        for (size_t i = 0; i < input_buffer_.size(); i++) out[i] = input_buffer_[i];
        return input_buffer_.size();
    }

   private:
    void duplexing() {
        for (size_t i = 0; i < input_buffer_.size(); i++) sponge_state_[i] = input_buffer_[i];
        input_buffer_.clear();
        gl_poseidon_permute_host(sponge_state_);
        output_buffer_.assign(sponge_state_, sponge_state_ + SPONGE_RATE);
    }
    F sponge_state_[SPONGE_WIDTH];
    std::vector<F> input_buffer_, output_buffer_;
};

// ---- FRI parameters (fri/mod.rs:30-143, reduction_strategies.rs:13-57) ----
struct FriReductionStrategy {
    enum Kind { Fixed, ConstantArityBits } kind = ConstantArityBits;
    std::vector<uint32_t> fixed;
    uint32_t arity_bits = 4, final_poly_bits = 5;
    std::vector<uint32_t> reduction_arity_bits(uint32_t degree_bits, uint32_t rate_bits, uint32_t cap_height) const {
        if (kind == Fixed) return fixed;
        std::vector<uint32_t> r;
        while (degree_bits > final_poly_bits && degree_bits + rate_bits - arity_bits >= cap_height) {
            r.push_back(arity_bits);
            degree_bits -= arity_bits;
        }
        return r;
    }
};
struct FriParams;
struct FriConfig {
    uint32_t rate_bits = 3, cap_height = 4, proof_of_work_bits = 16;
    FriReductionStrategy reduction_strategy;
    uint32_t num_query_rounds = 28;
    inline FriParams fri_params(uint32_t degree_bits, bool hiding) const;
    // CircuitConfig::standard_recursion_config().fri_config (plonk/circuit_data.rs:101-119)
    static FriConfig standard_recursion() { return FriConfig{}; }
};
struct FriParams {
    FriConfig config;
    bool hiding = false;
    uint32_t degree_bits = 0;
    std::vector<uint32_t> reduction_arity_bits;
    uint32_t lde_bits() const { return degree_bits + config.rate_bits; }
    size_t lde_size() const { return size_t(1) << lde_bits(); }
    size_t final_poly_len() const {
        uint32_t b = degree_bits;
        for (auto a : reduction_arity_bits) b -= a;
        return size_t(1) << b;
    }
};
inline FriParams FriConfig::fri_params(uint32_t degree_bits, bool hiding) const {
    return FriParams{*this, hiding, degree_bits, reduction_strategy.reduction_arity_bits(degree_bits, rate_bits, cap_height)};
}

// ---- FRI instance (fri/structure.rs:14-60) ----
struct FriPolynomialInfo {
    uint32_t oracle_index, polynomial_index;
};
struct FriBatchInfo {
    Ext point;
    std::vector<FriPolynomialInfo> polynomials;
};
struct FriOracleInfo {
    size_t num_polys;
    bool blinding;
};
struct FriInstanceInfo {
    std::vector<FriOracleInfo> oracles;
    std::vector<FriBatchInfo> batches;
};

// ---- FRI proof (fri/proof.rs:25-113) ----
struct FriQueryStep {
    std::vector<Ext> evals;
    MerkleProof merkle_proof;
};
struct FriInitialTreeProof {
    std::vector<std::pair<std::vector<F>, MerkleProof>> evals_proofs;
};
struct FriQueryRound {
    FriInitialTreeProof initial_trees_proof;
    std::vector<FriQueryStep> steps;
};
struct FriProof {
    std::vector<MerkleCap> commit_phase_merkle_caps;
    std::vector<FriQueryRound> query_round_proofs;
    std::vector<Ext> final_poly;
    F pow_witness = 0;
    // write_fri_proof (util/serialization/mod.rs:1595-1609): canonical little-endian u64s
    std::vector<uint8_t> to_bytes() const {
        std::vector<uint8_t> out;
        auto put = [&](F v) {
            for (int i = 0; i < 8; i++) out.push_back(uint8_t(v >> (8 * i)));
        };
        auto put_proof = [&](const MerkleProof& p) {
            out.push_back(uint8_t(p.siblings.size()));
            for (auto& h : p.siblings)
                for (F e : h.elements) put(e);
        };
        for (auto& cap : commit_phase_merkle_caps)
            for (auto& h : cap.hashes)
                for (F e : h.elements) put(e);
        for (auto& qr : query_round_proofs) {
            for (auto& ep : qr.initial_trees_proof.evals_proofs) {
                for (F e : ep.first) put(e);
                put_proof(ep.second);
            }
            for (auto& st : qr.steps) {
                for (auto& e : st.evals) {
                    put(e.c0);
                    put(e.c1);
                }
                put_proof(st.merkle_proof);
            }
        }
        for (auto& c : final_poly) {
            put(c.c0);
            put(c.c1);
        }
        put(pow_witness);
        return out;
    }
};

// The salt of a zero-knowledge commitment drawn on the device (gl_commit_finish_keyed): a 32-byte ChaCha20 key, which
// makes the commitment reproducible, or fresh entropy from the OS CSPRNG for each commitment (the reference's OsRng).
struct SaltKey {
    std::array<uint8_t, 32> key{};
    bool fresh = true;
    static SaltKey of(const std::array<uint8_t, 32>& k) {
        SaltKey s;
        s.key = k;
        s.fresh = false;
        return s;
    }
    static SaltKey os_entropy() { return SaltKey(); }
};

// ---- PolynomialBatch (fri/oracle.rs:30-237) ----
class PolynomialBatch {
   public:
    // from_values / from_coeffs with blinding and the salt drawn on the device from `key`
    static PolynomialBatch from_values(Context& ctx, const std::vector<std::vector<F>>& values, uint32_t rate_bits,
                                       bool blinding, uint32_t cap_height, const SaltKey& key) {
        return create_keyed(ctx, values, rate_bits, blinding, cap_height, key, false);
    }
    static PolynomialBatch from_coeffs(Context& ctx, const std::vector<std::vector<F>>& polynomials, uint32_t rate_bits,
                                       bool blinding, uint32_t cap_height, const SaltKey& key) {
        return create_keyed(ctx, polynomials, rate_bits, blinding, cap_height, key, true);
    }
    // from_values (oracle.rs:57-79): one Vec per polynomial; `salt` = SALT_SIZE columns of n << rate_bits
    // values when blinding (the reference draws them from OsRng).
    static PolynomialBatch from_values(Context& ctx, const std::vector<std::vector<F>>& values, uint32_t rate_bits,
                                       bool blinding, uint32_t cap_height, const std::vector<F>* salt = nullptr) {
        return create(ctx, values, rate_bits, blinding, cap_height, salt, false);
    }
    // from_coeffs (oracle.rs:82-112)
    static PolynomialBatch from_coeffs(Context& ctx, const std::vector<std::vector<F>>& polynomials, uint32_t rate_bits,
                                       bool blinding, uint32_t cap_height, const std::vector<F>* salt = nullptr) {
        return create(ctx, polynomials, rate_bits, blinding, cap_height, salt, true);
    }
    PolynomialBatch(PolynomialBatch&& o) noexcept { *this = std::move(o); }
    PolynomialBatch& operator=(PolynomialBatch&& o) noexcept {
        if (h_) gl_commit_destroy(h_);
        h_ = o.h_;
        ctx_ = o.ctx_;
        o.h_ = nullptr;
        return *this;
    }
    ~PolynomialBatch() {
        if (h_) gl_commit_destroy(h_);
    }
    gl_commit* handle() const { return h_; }
    Context& context() const { return *ctx_; }
    size_t num_polys() const { return gl_commit_num_polys(h_); }
    size_t leaf_width() const { return gl_commit_leaf_width(h_); }
    uint32_t degree_log() const { return gl_commit_degree_log(h_); }
    uint32_t rate_bits() const { return gl_commit_rate_bits(h_); }
    uint32_t cap_height() const { return gl_commit_cap_height(h_); }
    bool blinding() const { return leaf_width() != num_polys(); }
    // merkle_tree.cap
    MerkleCap cap() const {
        MerkleCap c;
        c.hashes.resize(size_t(1) << cap_height());
        check(gl_commit_cap(h_, c.hashes[0].elements, GL_MEM_HOST), ctx_->get());
        return c;
    }
    // polynomials[i].coeffs
    std::vector<std::vector<F>> polynomials() const {
        const size_t n = size_t(1) << degree_log(), B = num_polys();
        std::vector<F> flat(B * n);
        check(gl_commit_coeffs(h_, flat.data(), GL_MEM_HOST), ctx_->get());
        std::vector<std::vector<F>> out(B);
        for (size_t b = 0; b < B; b++) out[b].assign(flat.begin() + b * n, flat.begin() + (b + 1) * n);
        return out;
    }
    // get_lde_values(index, step) (oracle.rs:142-147)
    std::vector<F> get_lde_values(size_t index, size_t step) const {
        std::vector<F> v(num_polys());
        check(gl_commit_get_lde_values(h_, index, step, v.data()), ctx_->get());
        return v;
    }
    // merkle_tree.get(i) + merkle_tree.prove(i) for many indices
    void open(const std::vector<uint64_t>& idx, std::vector<std::vector<F>>& leaves, std::vector<MerkleProof>& proofs) const {
        const size_t W = leaf_width(), L = degree_log() + rate_bits() - cap_height();
        std::vector<F> lv(idx.size() * W), pt(idx.size() * L * 4 + 1);
        check(gl_commit_open(h_, idx.data(), idx.size(), lv.data(), pt.data()), ctx_->get());
        leaves.resize(idx.size());
        proofs.resize(idx.size());
        for (size_t q = 0; q < idx.size(); q++) {
            leaves[q].assign(lv.begin() + q * W, lv.begin() + (q + 1) * W);
            proofs[q].siblings.resize(L);
            if (L) std::memcpy(proofs[q].siblings[0].elements, &pt[q * L * 4], L * 32);
        }
    }
    // eval_commitment of OpeningSet::new (plonk/proof.rs:313-351)
    std::vector<Ext> eval_commitment(Ext z) const {
        std::vector<Ext> out(num_polys());
        F pt[2] = {z.c0, z.c1};
        check(gl_commit_eval_ext(h_, pt, &out[0].c0), ctx_->get());
        return out;
    }

    // OpeningSet::new / StarkOpeningSet::new (plonk/proof.rs:313-351, starky/src/proof.rs:221-260): every polynomial of
    // requests[i].first at requests[i].second, all in ONE native call (gl_openings); one vector of values per request.
    static std::vector<std::vector<Ext>> eval_commitments(const std::vector<std::pair<const PolynomialBatch*, Ext>>& requests) {
        std::vector<std::vector<Ext>> out(requests.size());
        if (requests.empty()) return out;
        Context& ctx = requests[0].first->context();
        std::vector<gl_commit*> handles;
        std::vector<uint32_t> pidx;
        std::vector<F> points;
        size_t total = 0;
        for (auto& rq : requests) {
            handles.push_back(rq.first->handle());
            size_t k = 0;
            for (; k < points.size() / 2; k++)
                if (points[2 * k] == rq.second.c0 && points[2 * k + 1] == rq.second.c1) break;
            if (k == points.size() / 2) {
                points.push_back(rq.second.c0);
                points.push_back(rq.second.c1);
            }
            pidx.push_back(uint32_t(k));
            total += rq.first->num_polys();
        }
        std::vector<Ext> flat(total);
        check(gl_openings(ctx.get(), handles.data(), pidx.data(), requests.size(), points.data(), points.size() / 2,
                          &flat[0].c0, GL_MEM_HOST), ctx.get());
        size_t off = 0;
        for (size_t i = 0; i < requests.size(); i++) {
            const size_t b = requests[i].first->num_polys();
            out[i].assign(flat.begin() + off, flat.begin() + off + b);
            off += b;
        }
        return out;
    }
    // compute_quotient_polys (plonk/prover.rs:609-815) from a recorded vanishing program (include/plonky2_b200.h,
    // gl_plonk_quotient; plonky2_b200/plonk.py builds such programs from gate lists): the LDEs of `commitments`
    // (constants_sigmas, wires, zs_partial_products[_lookup]) are read in place; returns num_challenges polynomials of
    // n << log2_ceil(quotient_degree_factor) coefficients in DEVICE memory at `out_coeffs_device`.
    static void compute_quotient_polys(const std::vector<const PolynomialBatch*>& commitments,
                                       const std::vector<gl_vp_instr>& program, const std::vector<F>& consts,
                                       const std::vector<F>& alphas, uint32_t num_vanishing_terms,
                                       uint32_t quotient_degree_factor, F* out_coeffs_device) {
        Context& ctx = commitments.at(0)->context();
        std::vector<gl_commit*> handles;
        for (auto* c : commitments) handles.push_back(c->handle());
        check(gl_plonk_quotient(ctx.get(), handles.data(), uint32_t(handles.size()), program.data(), uint32_t(program.size()),
                                consts.data(), uint32_t(consts.size()), alphas.data(), uint32_t(alphas.size()),
                                num_vanishing_terms, quotient_degree_factor, out_coeffs_device), ctx.get());
    }

    // The same commitment assembled from column groups that arrive over time (gl_commit_begin / add_columns / finish):
    // `kind` = GL_COLS_VALUES / GL_COLS_COEFFS / GL_COLS_COEFFS_CANONICAL, `mem` = GL_MEM_HOST / GL_MEM_DEVICE.
    static PolynomialBatch begin(Context& ctx, uint32_t num_polys, uint32_t degree_log, uint32_t rate_bits, uint32_t cap_height,
                                 uint32_t shard_index = 0, uint32_t num_shards = 1, F* coeff_storage = nullptr) {
        PolynomialBatch pb;
        pb.ctx_ = &ctx;
        check(gl_commit_begin(ctx.get(), num_polys, degree_log, rate_bits, cap_height, 0, shard_index, num_shards,
                              coeff_storage, &pb.h_), ctx.get());
        return pb;
    }
    void add_columns(uint32_t first_col, uint32_t count, const F* cols, size_t col_stride, int kind, int mem) {
        check(gl_commit_add_columns(h_, first_col, count, cols, col_stride, kind, mem), ctx_->get());
    }
    void finish() { check(gl_commit_finish(h_, nullptr, GL_MEM_HOST), ctx_->get()); }

    // prove_openings (oracle.rs:176-237) -> fri_proof (prover.rs:24-70): host transcript in the loop.
    static FriProof prove_openings(const FriInstanceInfo& instance, const std::vector<const PolynomialBatch*>& oracles,
                                   Challenger& challenger, const FriParams& fri_params) {
        Context& ctx = oracles.at(0)->context();
        const Ext alpha = challenger.get_extension_challenge();
        std::vector<gl_commit*> handles;
        for (auto* o : oracles) handles.push_back(o->handle());
        std::vector<gl_fri_batch> batches(instance.batches.size());
        std::vector<std::vector<uint32_t>> oi(batches.size()), pi(batches.size());
        for (size_t b = 0; b < batches.size(); b++) {
            for (auto& p : instance.batches[b].polynomials) {
                oi[b].push_back(p.oracle_index);
                pi[b].push_back(p.polynomial_index);
            }
            batches[b].point[0] = instance.batches[b].point.c0;
            batches[b].point[1] = instance.batches[b].point.c1;
            batches[b].num_polys = oi[b].size();
            batches[b].oracle_index = oi[b].data();
            batches[b].poly_index = pi[b].data();
        }
        const F al[2] = {alpha.c0, alpha.c1};
        gl_fri* f = nullptr;
        check(gl_fri_begin(ctx.get(), handles.data(), handles.size(), batches.data(), batches.size(), al,
                           fri_params.config.rate_bits, fri_params.config.cap_height, &f), ctx.get());
        std::unique_ptr<gl_fri, void (*)(gl_fri*)> guard(f, gl_fri_destroy);
        FriProof proof;
        // fri_committed_trees (prover.rs:84-150)
        const size_t C = size_t(1) << fri_params.config.cap_height;
        for (uint32_t arity_bits : fri_params.reduction_arity_bits) {
            MerkleCap cap;
            cap.hashes.resize(C);
            check(gl_fri_commit_round(f, arity_bits, cap.hashes[0].elements), ctx.get());
            challenger.observe_cap(cap);
            proof.commit_phase_merkle_caps.push_back(cap);
            const Ext beta = challenger.get_extension_challenge();
            const F be[2] = {beta.c0, beta.c1};
            check(gl_fri_fold(f, be), ctx.get());
        }
        proof.final_poly.resize(fri_params.final_poly_len());
        size_t len = 0;
        check(gl_fri_final_poly(f, &proof.final_poly[0].c0, 2 * proof.final_poly.size(), &len), ctx.get());
        proof.final_poly.resize(len);
        for (auto& c : proof.final_poly) challenger.observe_extension_element(c);
        // fri_proof_of_work (prover.rs:153-202)
        F st[12];
        const size_t pos = challenger.duplex_intermediate_state(st);
        check(gl_fri_pow(ctx.get(), st, (uint32_t)pos, fri_params.config.proof_of_work_bits, &proof.pow_witness), ctx.get());
        challenger.observe_element(proof.pow_witness);
        const F pow_response = challenger.get_challenge();
        if (fri_params.config.proof_of_work_bits && (pow_response >> (64 - fri_params.config.proof_of_work_bits)) != 0)
            throw Error(GL_ERR_POW_FAILED, "proof-of-work response does not have enough leading zeros");
        // fri_prover_query_rounds (prover.rs:204-258)
        const size_t nq = fri_params.config.num_query_rounds, n = fri_params.lde_size();
        std::vector<uint64_t> x(nq);
        for (auto& v : x) v = challenger.get_challenge() % n;
        proof.query_round_proofs.resize(nq);
        for (auto* o : oracles) {
            std::vector<std::vector<F>> leaves;
            std::vector<MerkleProof> proofs;
            o->open(x, leaves, proofs);
            for (size_t q = 0; q < nq; q++)
                proof.query_round_proofs[q].initial_trees_proof.evals_proofs.emplace_back(leaves[q], proofs[q]);
        }
        std::vector<uint64_t> cur = x;
        uint32_t log_cur = fri_params.lde_bits();
        for (size_t r = 0; r < fri_params.reduction_arity_bits.size(); r++) {
            const uint32_t ab = fri_params.reduction_arity_bits[r];
            for (auto& v : cur) v >>= ab;
            const size_t W = size_t(2) << ab, L = log_cur - ab - fri_params.config.cap_height;
            std::vector<F> lv(nq * W), pt(nq * L * 4 + 1);
            check(gl_fri_open(f, (uint32_t)r, cur.data(), nq, lv.data(), pt.data()), ctx.get());
            for (size_t q = 0; q < nq; q++) {
                FriQueryStep st2;
                st2.evals.resize(W / 2);
                std::memcpy(&st2.evals[0].c0, &lv[q * W], W * 8);
                st2.merkle_proof.siblings.resize(L);
                if (L) std::memcpy(st2.merkle_proof.siblings[0].elements, &pt[q * L * 4], L * 32);
                proof.query_round_proofs[q].steps.push_back(std::move(st2));
            }
            log_cur -= ab;
        }
        return proof;
    }

   private:
    PolynomialBatch() = default;
    static PolynomialBatch create(Context& ctx, const std::vector<std::vector<F>>& cols, uint32_t rate_bits, bool blinding,
                                  uint32_t cap_height, const std::vector<F>* salt, bool is_coeffs) {
        if (cols.empty()) throw ShapeError(GL_ERR_BAD_SHAPE, "empty polynomial batch");
        const size_t n = cols[0].size();
        const uint32_t log_n = log2_strict(n);
        std::vector<F> flat(cols.size() * n);
        for (size_t b = 0; b < cols.size(); b++) {
            if (cols[b].size() != n) throw ShapeError(GL_ERR_BAD_SHAPE, "Polynomial degrees inconsistent");  // oracle.rs:128
            std::memcpy(&flat[b * n], cols[b].data(), n * 8);
        }
        if (blinding && (!salt || salt->size() != SALT_SIZE * (n << rate_bits)))
            throw ShapeError(GL_ERR_BAD_SHAPE, "blinding needs SALT_SIZE * (n << rate_bits) salt values");
        PolynomialBatch pb;
        pb.ctx_ = &ctx;
        check(gl_commit_create(ctx.get(), flat.data(), n, (uint32_t)cols.size(), log_n, rate_bits, cap_height,
                               blinding ? salt->data() : nullptr, is_coeffs ? 1 : 0, GL_MEM_HOST, &pb.h_), ctx.get());
        return pb;
    }
    // gl_commit_begin -> gl_commit_add_columns -> gl_commit_finish_keyed
    static PolynomialBatch create_keyed(Context& ctx, const std::vector<std::vector<F>>& cols, uint32_t rate_bits,
                                        bool blinding, uint32_t cap_height, const SaltKey& key, bool is_coeffs) {
        if (!blinding) throw ShapeError(GL_ERR_BAD_SHAPE, "a salt key needs blinding");
        if (cols.empty()) throw ShapeError(GL_ERR_BAD_SHAPE, "empty polynomial batch");
        const size_t n = cols[0].size();
        const uint32_t log_n = log2_strict(n);
        std::vector<F> flat(cols.size() * n);
        for (size_t b = 0; b < cols.size(); b++) {
            if (cols[b].size() != n) throw ShapeError(GL_ERR_BAD_SHAPE, "Polynomial degrees inconsistent");  // oracle.rs:128
            std::memcpy(&flat[b * n], cols[b].data(), n * 8);
        }
        PolynomialBatch pb;
        pb.ctx_ = &ctx;
        check(gl_commit_begin(ctx.get(), (uint32_t)cols.size(), log_n, rate_bits, cap_height, 1, 0, 1, nullptr, &pb.h_),
              ctx.get());
        check(gl_commit_add_columns(pb.h_, 0, (uint32_t)cols.size(), flat.data(), n,
                                    is_coeffs ? GL_COLS_COEFFS : GL_COLS_VALUES, GL_MEM_HOST), ctx.get());
        check(gl_commit_finish_keyed(pb.h_, key.fresh ? nullptr : key.key.data()), ctx.get());
        return pb;
    }
    gl_commit* h_ = nullptr;
    Context* ctx_ = nullptr;
};

}  // namespace plonky2_b200
