// gl_oracle.cpp -- CPU parity oracle (TEST INFRASTRUCTURE ONLY; see gl_oracle.h header comment).
//
// A deliberately plain restatement of the reference CPU algorithm. It follows the reference's
// control flow (bit-reverse + radix-2 DIT NTT, per-column LDE, transpose + row bit-reversal,
// recursive Merkle fill, coefficient-domain FRI fold + re-FFT) so that it is an independent
// check of the GPU path, which uses different algorithms (four-step NTT, coset-wise LDE,
// level-order Merkle build, value-domain leaf-local FRI fold).
#include "gl_oracle.h"

#include <algorithm>
#include <cassert>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <sys/mman.h>

#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

#include "gl_poseidon_constants.h"

typedef unsigned __int128 u128;
typedef uint64_t u64;

namespace {

// ------------------------------------------------------------------ parallelism (stands in for rayon)
// A persistent worker pool with dynamically scheduled chunks: the reference runs its par_iter / join calls on
// rayon's global pool (maybe_rayon/src/lib.rs), which neither respawns threads per call nor splits statically.
class Pool {
   public:
    static Pool& get() {
        static Pool p;
        return p;
    }
    // run job(chunk_index) for chunk_index < nchunks on up to `nthreads` threads (the caller is one of them)
    void run(size_t nchunks, int nthreads, const std::function<void(size_t)>& job) {
        if (nthreads <= 1 || nchunks <= 1) {
            for (size_t i = 0; i < nchunks; i++) job(i);
            return;
        }
        std::unique_lock<std::mutex> api(api_mu_);  // one parallel region at a time (no nesting in this file)
        ensure(nthreads - 1);
        {
            std::lock_guard<std::mutex> lk(mu_);
            job_ = &job;
            nchunks_ = nchunks;
            next_.store(0);
            active_ = std::min<size_t>(workers_.size(), (size_t)nthreads - 1);
            pending_ = active_;
            epoch_++;
        }
        cv_.notify_all();
        work();
        std::unique_lock<std::mutex> lk(mu_);
        done_cv_.wait(lk, [&] { return pending_ == 0; });
        job_ = nullptr;
    }
    ~Pool() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
            epoch_++;
        }
        cv_.notify_all();
        for (auto& t : workers_) t.join();
    }

   private:
    void work() {
        for (;;) {
            size_t i = next_.fetch_add(1);
            if (i >= nchunks_) break;
            (*job_)(i);
        }
    }
    void ensure(size_t n) {
        while (workers_.size() < n) {
            size_t id = workers_.size();
            workers_.emplace_back([this, id] {
                size_t seen = 0;
                for (;;) {
                    std::unique_lock<std::mutex> lk(mu_);
                    cv_.wait(lk, [&] { return stop_ || (epoch_ != seen && id < active_); });
                    if (stop_) return;
                    seen = epoch_;
                    lk.unlock();
                    work();
                    lk.lock();
                    if (--pending_ == 0) done_cv_.notify_all();
                }
            });
        }
    }
    std::mutex api_mu_, mu_;
    std::condition_variable cv_, done_cv_;
    std::vector<std::thread> workers_;
    const std::function<void(size_t)>* job_ = nullptr;
    std::atomic<size_t> next_{0};
    size_t nchunks_ = 0, active_ = 0, pending_ = 0, epoch_ = 0;
    bool stop_ = false;
};
// f(i) for i < n, in chunks of `grain` consecutive indices
template <class F>
void parallel_for(size_t n, int nthreads, F f, size_t grain = 1) {
    if (grain < 1) grain = 1;
    const size_t nchunks = (n + grain - 1) / grain;
    Pool::get().run(nchunks, nthreads, [&](size_t c) {
        const size_t lo = c * grain, hi = std::min(n, lo + grain);
        for (size_t i = lo; i < hi; i++) f(i);
    });
}

// Uninitialised storage (Rust's Vec::with_capacity + set_len / collect: no serial zero-fill, pages are first
// touched by the threads that write them). Large blocks are recycled through a small free list, like the
// reference's allocator (jemalloc/system malloc keep freed arenas mapped): without it every call re-faults
// gigabytes of fresh pages, which serialises on the kernel's mm lock when 128 threads touch them at once.
struct BlockCache {
    static const size_t MIN_BYTES = (size_t)1 << 20, MAX_BLOCKS = 8;
    std::mutex mu;
    std::vector<std::pair<size_t, void*>> free_blocks;
    void* get(size_t bytes) {
        if (bytes >= MIN_BYTES) {
            std::lock_guard<std::mutex> lk(mu);
            size_t best = free_blocks.size();
            for (size_t i = 0; i < free_blocks.size(); i++)
                if (free_blocks[i].first >= bytes && free_blocks[i].first <= bytes + bytes / 4 &&
                    (best == free_blocks.size() || free_blocks[i].first < free_blocks[best].first))
                    best = i;
            if (best != free_blocks.size()) {
                void* q = free_blocks[best].second;
                free_blocks.erase(free_blocks.begin() + best);
                return q;
            }
        }
        void* q = nullptr;
        if (bytes >= MIN_BYTES) {
            if (posix_memalign(&q, (size_t)2 << 20, bytes) != 0) q = nullptr;
#if defined(MADV_HUGEPAGE)
            if (q) madvise(q, bytes, MADV_HUGEPAGE);
#endif
        } else {
            q = malloc(bytes);
        }
        return q;
    }
    void put(void* q, size_t bytes) {
        if (!q) return;
        if (bytes >= MIN_BYTES) {
            std::lock_guard<std::mutex> lk(mu);
            if (free_blocks.size() < MAX_BLOCKS) {
                free_blocks.emplace_back(bytes, q);
                return;
            }
            // evict the smallest cached block in favour of a larger one
            size_t sm = 0;
            for (size_t i = 1; i < free_blocks.size(); i++)
                if (free_blocks[i].first < free_blocks[sm].first) sm = i;
            if (free_blocks[sm].first < bytes) {
                free(free_blocks[sm].second);
                free_blocks[sm] = std::make_pair(bytes, q);
                return;
            }
        }
        free(q);
    }
    static BlockCache& get_cache() {
        static BlockCache* c = new BlockCache();  // leaked on purpose: blocks may outlive static destruction order
        return *c;
    }
};
template <class T>
struct RawVec {
    T* p = nullptr;
    size_t n = 0;
    RawVec() {}
    RawVec(const RawVec&) = delete;
    RawVec& operator=(const RawVec&) = delete;
    ~RawVec() { BlockCache::get_cache().put(p, n * sizeof(T)); }
    void resize(size_t m) {
        BlockCache::get_cache().put(p, n * sizeof(T));
        p = m ? (T*)BlockCache::get_cache().get(m * sizeof(T)) : nullptr;
        if (m && !p) {
            fprintf(stderr, "oracle: out of memory (%zu bytes)\n", m * sizeof(T));
            abort();
        }
        n = m;
    }
    void clear() { resize(0); }
    T* data() { return p; }
    const T* data() const { return p; }
    size_t size() const { return n; }
    T& operator[](size_t i) { return p[i]; }
    const T& operator[](size_t i) const { return p[i]; }
    T* begin() { return p; }
    T* end() { return p + n; }
    const T* begin() const { return p; }
    const T* end() const { return p + n; }
};

// ------------------------------------------------------------------ field
// field/src/goldilocks_field.rs:13-25,198
const u64 P = 0xFFFFFFFF00000001ULL;
const u64 EPS = 0xFFFFFFFFULL;
// field/src/goldilocks_field.rs:80,87,76
const u64 MULTIPLICATIVE_GROUP_GENERATOR = 14293326489335486720ULL;
const u64 POWER_OF_TWO_GENERATOR = 7277203076849721926ULL;
const uint32_t TWO_ADICITY = 32;

// to_canonical_u64, goldilocks_field.rs:216-224
inline u64 canon(u64 c) { return c >= P ? c - P : c; }

// Add, goldilocks_field.rs:245-267
inline u64 fadd(u64 a, u64 b) {
    u64 sum = a + b;
    bool over = sum < a;
    u64 sum2 = sum + ((0 - (u64)over) & EPS);
    bool over2 = sum2 < sum;
    if (over2) sum2 += EPS;
    return sum2;
}
// Sub, goldilocks_field.rs:282-304
inline u64 fsub(u64 a, u64 b) {
    u64 diff = a - b;
    bool under = a < b;
    u64 diff2 = diff - ((0 - (u64)under) & EPS);
    bool under2 = diff2 > diff;
    if (under2) diff2 -= EPS;
    return diff2;
}
// reduce128, goldilocks_field.rs:401-415 (+ add_no_canonicalize_trashing_input :355-389)
inline u64 reduce128(u128 x) {
    u64 x_lo = (u64)x, x_hi = (u64)(x >> 64);
    u64 x_hi_hi = x_hi >> 32;
    u64 x_hi_lo = x_hi & EPS;
    u64 t0 = x_lo - x_hi_hi;
    if (x_lo < x_hi_hi) t0 -= EPS;
    u64 t1 = x_hi_lo * EPS;
    u64 res = t0 + t1;
    // add_no_canonicalize_trashing_input (:355-389): branch-free "+= EPS * carry" (the carry is ~50% likely)
    res += (0 - (u64)(res < t0)) & EPS;
    return res;
}
// Mul, goldilocks_field.rs:313-320
inline u64 fmul(u64 a, u64 b) { return reduce128((u128)a * (u128)b); }
inline u64 fsqr(u64 a) { return fmul(a, a); }
inline u64 fneg(u64 a) {
    u64 c = canon(a);
    return c == 0 ? 0 : P - c;
}
// exp_u64 (types.rs:359-376): square-and-multiply
u64 fexp(u64 base, u64 e) {
    u64 cur = base, prod = 1;
    while (e) {
        if (e & 1) prod = fmul(prod, cur);
        cur = fsqr(cur);
        e >>= 1;
    }
    return prod;
}
// try_inverse = a^(p-2) (goldilocks_field.rs:108-147; any addition chain gives the same value)
u64 finv(u64 a) { return canon(a) == 0 ? 0 : fexp(a, P - 2); }
// primitive_root_of_unity, types.rs:268-272
u64 primitive_root_of_unity(uint32_t n_log) {
    assert(n_log <= TWO_ADICITY);
    u64 b = POWER_OF_TWO_GENERATOR;
    for (uint32_t i = 0; i < TWO_ADICITY - n_log; i++) b = fsqr(b);
    return b;
}
// inverse_2exp, types.rs:226-266 : for exp <= two_adicity, 2^-k = p - (p-1)/2^k
u64 inverse_2exp(uint32_t k) {
    if (k <= TWO_ADICITY) return P - ((P - 1) >> k);
    return finv(fexp(2, k));
}

// ------------------------------------------------------------------ quadratic extension
// goldilocks_extensions.rs:14-27 (W = 7), extension/quadratic.rs:180-193
struct E2 {
    u64 a, b;
};
inline E2 e2(u64 a, u64 b = 0) { return E2{a, b}; }
inline E2 eadd(E2 x, E2 y) { return E2{fadd(x.a, y.a), fadd(x.b, y.b)}; }
inline E2 esub(E2 x, E2 y) { return E2{fsub(x.a, y.a), fsub(x.b, y.b)}; }
inline E2 emul(E2 x, E2 y) {
    u64 c0 = fadd(fmul(x.a, y.a), fmul(7, fmul(x.b, y.b)));
    u64 c1 = fadd(fmul(x.a, y.b), fmul(x.b, y.a));
    return E2{c0, c1};
}
inline E2 escale(E2 x, u64 s) { return E2{fmul(x.a, s), fmul(x.b, s)}; }
// try_inverse, extension/quadratic.rs:86-100: a^-1 = frob(a) / (a * frob(a)), frob = conjugation
E2 einv(E2 x) {
    u64 norm = fsub(fsqr(x.a), fmul(7, fsqr(x.b)));
    u64 ninv = finv(norm);
    return E2{fmul(x.a, ninv), fmul(fneg(x.b), ninv)};
}
inline bool eeq(E2 x, E2 y) { return canon(x.a) == canon(y.a) && canon(x.b) == canon(y.b); }
E2 eexp(E2 base, u64 e) {
    E2 cur = base, prod = e2(1);
    while (e) {
        if (e & 1) prod = emul(prod, cur);
        cur = emul(cur, cur);
        e >>= 1;
    }
    return prod;
}

// ------------------------------------------------------------------ bit reversal
uint32_t log2_strict(size_t n) {
    uint32_t l = 0;
    while (((size_t)1 << l) < n) l++;
    if (((size_t)1 << l) != n) {
        fprintf(stderr, "oracle: Not a power of two: %zu\n", n);  // util/src/lib.rs:28
        abort();
    }
    return l;
}
// reverse_bits, plonky2/src/util/mod.rs:33-41
inline u64 reverse_bits(u64 x, uint32_t bits) {
    u64 r = 0;
    for (uint32_t i = 0; i < bits; i++) r |= ((x >> i) & 1) << (bits - 1 - i);
    return r;
}
// reverse_index_bits_in_place, util/src/lib.rs:185-234 (semantics: arr[i] <-> arr[bitrev(i)])
void reverse_index_bits_in_place(u64* arr, size_t n, size_t w) {
    uint32_t lg = log2_strict(n);
    std::vector<u64> tmp(w);
    for (size_t i = 0; i < n; i++) {
        size_t j = reverse_bits(i, lg);
        if (i < j) {
            if (w == 1) {
                std::swap(arr[i], arr[j]);
            } else {
                memcpy(tmp.data(), arr + i * w, w * 8);
                memcpy(arr + i * w, arr + j * w, w * 8);
                memcpy(arr + j * w, tmp.data(), w * 8);
            }
        }
    }
}

// ------------------------------------------------------------------ NTT
// fft_root_table, field/src/fft.rs:14-33
typedef std::vector<std::vector<u64>> RootTable;
RootTable fft_root_table(size_t n) {
    uint32_t lg_n = log2_strict(n);
    std::vector<u64> bases;
    u64 base = primitive_root_of_unity(lg_n);
    bases.push_back(base);
    for (uint32_t i = 1; i < lg_n; i++) {
        base = fsqr(base);
        bases.push_back(base);
    }
    RootTable t;
    for (uint32_t lg_m = 1; lg_m <= lg_n; lg_m++) {
        size_t half_m = (size_t)1 << (lg_m - 1);
        u64 b = bases[lg_n - lg_m];
        size_t cnt = std::max(half_m, (size_t)2);
        std::vector<u64> row(cnt);
        u64 cur = 1;
        for (size_t i = 0; i < cnt; i++) {
            row[i] = cur;
            cur = fmul(cur, b);
        }
        t.push_back(std::move(row));
    }
    return t;
}
// fft_classic (+ scalar fft_classic_simd), field/src/fft.rs:95-202
void fft_classic(u64* values, size_t n, uint32_t r, const RootTable& root_table) {
    reverse_index_bits_in_place(values, n, 1);
    uint32_t lg_n = log2_strict(n);
    if (root_table.size() != lg_n) {
        fprintf(stderr, "oracle: Expected root table of length %u, but it was %zu.\n", lg_n,
                root_table.size());
        abort();
    }
    if (r > 0) {
        size_t mask = ~(((size_t)1 << r) - 1);
        for (size_t i = 0; i < n; i++) values[i] = values[i & mask];
    }
    for (uint32_t lg_half_m = r; lg_half_m < lg_n; lg_half_m++) {
        size_t m = (size_t)1 << (lg_half_m + 1);
        size_t half_m = m / 2;
        const std::vector<u64>& omega_table = root_table[lg_half_m];
        for (size_t k = 0; k < n; k += m) {
            for (size_t j = 0; j < half_m; j++) {
                u64 omega = omega_table[j];
                u64 t = fmul(omega, values[k + half_m + j]);
                u64 u = values[k + j];
                values[k + j] = fadd(u, t);
                values[k + half_m + j] = fsub(u, t);
            }
        }
    }
}
// fft_with_options, fft.rs:53-61
void fft_with_options(u64* buf, size_t n, uint32_t zero_factor, const RootTable* rt) {
    if (n == 1) return;
    if (rt) {
        fft_classic(buf, n, zero_factor, *rt);
    } else {
        RootTable t = fft_root_table(n);
        fft_classic(buf, n, zero_factor, t);
    }
}
// ifft_with_options, fft.rs:68-91
void ifft_with_options(u64* buf, size_t n, const RootTable* rt) {
    uint32_t lg_n = log2_strict(n);
    u64 n_inv = inverse_2exp(lg_n);
    fft_with_options(buf, n, 0, rt);
    if (n == 1) return;
    buf[0] = fmul(buf[0], n_inv);
    buf[n / 2] = fmul(buf[n / 2], n_inv);
    for (size_t i = 1; i < n / 2; i++) {
        size_t j = n - i;
        u64 ci = fmul(buf[j], n_inv);
        u64 cj = fmul(buf[i], n_inv);
        buf[i] = ci;
        buf[j] = cj;
    }
}
// coset_fft_with_options, polynomial/mod.rs:280-293
void coset_fft_with_options(u64* buf, size_t n, u64 shift, uint32_t zero_factor, const RootTable* rt) {
    u64 r = 1;
    for (size_t i = 0; i < n; i++) {
        buf[i] = fmul(r, buf[i]);
        r = fmul(r, shift);
    }
    fft_with_options(buf, n, zero_factor, rt);
}
// coset_ifft, polynomial/mod.rs:63-73
void coset_ifft(u64* buf, size_t n, u64 shift) {
    ifft_with_options(buf, n, nullptr);
    u64 sinv = finv(shift), r = 1;
    for (size_t i = 0; i < n; i++) {
        buf[i] = fmul(buf[i], r);
        r = fmul(r, sinv);
    }
}

// ------------------------------------------------------------------ Poseidon
// constant_layer, poseidon.rs:630-641
inline void constant_layer(u64 st[12], int round_ctr) {
    for (int i = 0; i < 12; i++) st[i] = fadd(st[i], GL_POSEIDON_RC[i + 12 * round_ctr]);
}
// sbox_monomial, poseidon.rs:689-696
inline u64 sbox(u64 x) {
    u64 x2 = fsqr(x), x4 = fsqr(x2), x3 = fmul(x, x2);
    return fmul(x3, x4);
}
// mds_row_shf + mds_layer, poseidon.rs:180-200,269-290 -- evaluated like the reference's Goldilocks
// override (poseidon_goldilocks.rs:217-248) on the low/high 32-bit halves of the state so that the
// 12-term sums of (32-bit x 6-bit) products fit in u64 and one reduction per lane suffices.
inline void mds_layer(u64 st[12]) {
    u64 lo[24], hi[24];
    for (int i = 0; i < 12; i++) {
        lo[i] = lo[i + 12] = st[i] & EPS;
        hi[i] = hi[i + 12] = st[i] >> 32;
    }
    for (int r = 0; r < 12; r++) {
        u64 al = 0, ah = 0;
        for (int i = 0; i < 12; i++) {
            al += lo[i + r] * GL_POSEIDON_MDS_CIRC[i];
            ah += hi[i + r] * GL_POSEIDON_MDS_CIRC[i];
        }
        al += lo[r] * GL_POSEIDON_MDS_DIAG[r];
        ah += hi[r] * GL_POSEIDON_MDS_DIAG[r];
        u128 sum = (u128)al + ((u128)ah << 32);
        st[r] = reduce128(sum);
    }
}
// full_rounds, poseidon.rs:741-749
inline void full_rounds(u64 st[12], int* round_ctr) {
    for (int k = 0; k < GL_POSEIDON_HALF_FULL_ROUNDS; k++) {
        constant_layer(st, *round_ctr);
        for (int i = 0; i < 12; i++) st[i] = sbox(st[i]);
        mds_layer(st);
        (*round_ctr)++;
    }
}
// u160 accumulator of 64x64 products and its reduction (poseidon.rs:40-53: add_u160_u128, reduce_u160)
struct U160 {
    u128 lo;
    uint32_t hi;
};
inline void add_u160_u128(U160& x, u128 y) {
    x.lo += y;
    x.hi += (uint32_t)(x.lo < y);
}
// reduce96 / from_noncanonical_u96, goldilocks_field.rs:159-161,392-398
inline u64 reduce96(u64 n_lo, uint32_t n_hi) {
    u64 t1 = (u64)n_hi * EPS;
    u64 res = n_lo + t1;
    res += (0 - (u64)(res < t1)) & EPS;
    return res;
}
inline u64 reduce_u160(const U160& x) {
    u64 reduced_hi = reduce96((u64)(x.lo >> 64), x.hi);
    return reduce128(((u128)reduced_hi << 64) + (u128)(u64)x.lo);
}
// mds_partial_layer_init, poseidon.rs:413-441. The reference accumulates result[c] += state[r] * t in the field;
// the sums are evaluated here in a u160 accumulator with ONE reduction per output lane (same field value).
inline void mds_partial_layer_init(u64 st[12]) {
    u64 result[12];
    result[0] = st[0];
    for (int c = 1; c < 12; c++) {
        U160 acc = {0, 0};
        for (int r = 1; r < 12; r++) add_u160_u128(acc, (u128)st[r] * GL_POSEIDON_FAST_INIT_MATRIX[(r - 1) * 11 + (c - 1)]);
        result[c] = reduce_u160(acc);
    }
    memcpy(st, result, sizeof(result));
}
// mds_partial_layer_fast, poseidon.rs:514-542: u160 accumulator for d, multiply_accumulate for the other lanes
// (goldilocks_field.rs:118-123: reduce128(a*b + c))
inline void mds_partial_layer_fast(u64 st[12], int r) {
    U160 d_sum = {0, 0};
    for (int i = 1; i < 12; i++) add_u160_u128(d_sum, (u128)st[i] * GL_POSEIDON_FAST_W_HATS[r * 11 + i - 1]);
    add_u160_u128(d_sum, (u128)st[0] * (GL_POSEIDON_MDS_CIRC[0] + GL_POSEIDON_MDS_DIAG[0]));
    u64 result[12];
    result[0] = reduce_u160(d_sum);
    for (int i = 1; i < 12; i++)
        result[i] = reduce128((u128)st[0] * GL_POSEIDON_FAST_VS[r * 11 + i - 1] + (u128)st[i]);
    memcpy(st, result, sizeof(result));
}
// partial_rounds, poseidon.rs:751-764
inline void partial_rounds(u64 st[12], int* round_ctr) {
    for (int i = 0; i < 12; i++) st[i] = fadd(st[i], GL_POSEIDON_FAST_FIRST_RC[i]);
    mds_partial_layer_init(st);
    for (int i = 0; i < GL_POSEIDON_PARTIAL_ROUNDS; i++) {
        st[0] = sbox(st[0]);
        st[0] = fadd(st[0], GL_POSEIDON_FAST_RC[i]);
        mds_partial_layer_fast(st, i);
    }
    *round_ctr += GL_POSEIDON_PARTIAL_ROUNDS;
}
// poseidon, poseidon.rs:766-777
void poseidon(u64 st[12]) {
    int round_ctr = 0;
    full_rounds(st, &round_ctr);
    partial_rounds(st, &round_ctr);
    full_rounds(st, &round_ctr);
    assert(round_ctr == GL_POSEIDON_ROUNDS);
}
// poseidon_naive, poseidon.rs:779-801
void poseidon_naive(u64 st[12]) {
    int round_ctr = 0;
    full_rounds(st, &round_ctr);
    for (int k = 0; k < GL_POSEIDON_PARTIAL_ROUNDS; k++) {
        constant_layer(st, round_ctr);
        st[0] = sbox(st[0]);
        mds_layer(st);
        round_ctr++;
    }
    full_rounds(st, &round_ctr);
}

struct Hash {
    u64 e[4];
};
// hash_n_to_m_no_pad (num_outputs = 4), hashing.rs:118-145 (overwrite-mode sponge, rate 8)
Hash hash_no_pad(const u64* in, size_t len) {
    u64 st[12] = {0};
    for (size_t off = 0; off < len; off += 8) {
        size_t c = std::min((size_t)8, len - off);
        for (size_t i = 0; i < c; i++) st[i] = in[off + i];
        poseidon(st);
    }
    Hash h;
    for (int i = 0; i < 4; i++) h.e[i] = canon(st[i]);
    return h;
}
// hash_or_noop, plonk/config.rs:63-74
Hash hash_or_noop(const u64* in, size_t len) {
    if (len * 8 <= 32) {
        Hash h = {{0, 0, 0, 0}};
        for (size_t i = 0; i < len; i++) h.e[i] = canon(in[i]);
        return h;
    }
    return hash_no_pad(in, len);
}
// compress / two_to_one, hashing.rs:97-114, poseidon.rs:884-886
Hash two_to_one(const Hash& l, const Hash& r) {
    u64 st[12] = {l.e[0], l.e[1], l.e[2], l.e[3], r.e[0], r.e[1], r.e[2], r.e[3], 0, 0, 0, 0};
    poseidon(st);
    Hash h;
    for (int i = 0; i < 4; i++) h.e[i] = canon(st[i]);
    return h;
}
inline bool heq(const Hash& a, const Hash& b) { return memcmp(a.e, b.e, 32) == 0; }

// ------------------------------------------------------------------ Merkle tree
// fill_subtree, merkle_tree.rs:86-113. digests_buf has 2*(n_leaves-1) hashes.
Hash fill_subtree(Hash* digests_buf, size_t buf_len, const u64* leaves, size_t n_leaves, size_t W) {
    assert(n_leaves == buf_len / 2 + 1);
    if (buf_len == 0) return hash_or_noop(leaves, W);
    size_t half = buf_len / 2;
    Hash* left_buf = digests_buf;           // [0, half-1)
    Hash* left_digest_mem = digests_buf + half - 1;
    Hash* right_digest_mem = digests_buf + half;
    Hash* right_buf = digests_buf + half + 1;
    size_t sub_len = half - 1;
    size_t nl = n_leaves / 2;
    Hash ld = fill_subtree(left_buf, sub_len, leaves, nl, W);
    Hash rd = fill_subtree(right_buf, sub_len, leaves + nl * W, nl, W);
    *left_digest_mem = ld;
    *right_digest_mem = rd;
    return two_to_one(ld, rd);
}
// rayon::join of the recursion (merkle_tree.rs:100-104) as pool tasks: the subtrees `depth` levels down are the
// tasks; the few nodes above them are combined afterwards in the same recursive order.
struct SubTask {
    Hash* buf;
    size_t buf_len;
    const u64* leaves;
    size_t n_leaves;
    Hash out;
};
void collect_subtasks(Hash* buf, size_t buf_len, const u64* leaves, size_t n_leaves, size_t W, int depth,
                      std::vector<SubTask>& tasks) {
    if (depth == 0 || buf_len == 0) {
        tasks.push_back(SubTask{buf, buf_len, leaves, n_leaves, Hash()});
        return;
    }
    size_t half = buf_len / 2, sub_len = half - 1, nl = n_leaves / 2;
    collect_subtasks(buf, sub_len, leaves, nl, W, depth - 1, tasks);
    collect_subtasks(buf + half + 1, sub_len, leaves + nl * W, nl, W, depth - 1, tasks);
}
Hash combine_subtasks(Hash* buf, size_t buf_len, int depth, const SubTask*& it) {
    if (depth == 0 || buf_len == 0) return (it++)->out;
    size_t half = buf_len / 2, sub_len = half - 1;
    Hash ld = combine_subtasks(buf, sub_len, depth - 1, it);
    Hash rd = combine_subtasks(buf + half + 1, sub_len, depth - 1, it);
    buf[half - 1] = ld;
    buf[half] = rd;
    return two_to_one(ld, rd);
}
// MerkleTree::new + fill_digests_buf, merkle_tree.rs:115-149,193-224
int merkle_build(const u64* leaves, size_t N, size_t W, uint32_t cap_height, Hash* digests, Hash* cap,
                 int nthreads) {
    uint32_t lg = log2_strict(N);
    if (cap_height > lg) {
        fprintf(stderr, "oracle: cap_height=%u should be at most log2(leaves.len())=%u\n", cap_height, lg);
        return 1;
    }
    size_t C = (size_t)1 << cap_height;
    size_t num_digests = 2 * (N - C);
    if (nthreads < 1) nthreads = 1;
    if (num_digests == 0) {
        parallel_for(N, nthreads, [&](size_t i) { cap[i] = hash_or_noop(leaves + i * W, W); }, 64);
        return 0;
    }
    size_t sub_digests = num_digests >> cap_height;
    size_t sub_leaves = N >> cap_height;
    // one task per cap subtree (par_chunks), recursive join inside: split until there are ~8 tasks per thread
    int depth = 0;
    while (((size_t)C << depth) < (size_t)nthreads * 8 && ((size_t)1 << (depth + 1)) <= sub_leaves / 2) depth++;
    std::vector<SubTask> tasks;
    for (size_t c = 0; c < C; c++)
        collect_subtasks(digests + c * sub_digests, sub_digests, leaves + c * sub_leaves * W, sub_leaves, W, depth, tasks);
    parallel_for(tasks.size(), nthreads, [&](size_t t) {
        SubTask& k = tasks[t];
        k.out = fill_subtree(k.buf, k.buf_len, k.leaves, k.n_leaves, W);
    });
    const SubTask* it = tasks.data();
    for (size_t c = 0; c < C; c++) cap[c] = combine_subtasks(digests + c * sub_digests, sub_digests, depth, it);
    return 0;
}
// merkle_tree_prove, merkle_tree.rs:151-190
void merkle_prove(size_t leaf_index, size_t leaves_len, uint32_t cap_height, const Hash* digests,
                  Hash* out) {
    uint32_t num_layers = log2_strict(leaves_len) - cap_height;
    size_t digest_len = 2 * (leaves_len - ((size_t)1 << cap_height));
    size_t tree_index = leaf_index >> num_layers;
    size_t tree_len = digest_len >> cap_height;
    const Hash* digest_tree = digests + tree_len * tree_index;
    size_t pair_index = leaf_index & (((size_t)1 << num_layers) - 1);
    for (uint32_t i = 0; i < num_layers; i++) {
        size_t parity = pair_index & 1;
        pair_index >>= 1;
        size_t siblings_index = (pair_index << (i + 1)) + ((size_t)1 << i) - 1;
        size_t sibling_index = 2 * siblings_index + (1 - parity);
        out[i] = digest_tree[sibling_index];
    }
}
// verify_merkle_proof_to_cap, merkle_proofs.rs:55-107 (single leaf)
bool merkle_verify(const u64* leaf, size_t W, size_t leaf_index, const Hash* siblings, size_t n_sib,
                   const Hash* cap) {
    Hash cur = hash_or_noop(leaf, W);
    for (size_t i = 0; i < n_sib; i++) {
        size_t bit = leaf_index & 1;
        leaf_index >>= 1;
        cur = bit ? two_to_one(siblings[i], cur) : two_to_one(cur, siblings[i]);
    }
    return heq(cur, cap[leaf_index]);
}

}  // namespace

// ------------------------------------------------------------------ PolynomialBatch
struct glo_commit {
    size_t B, W, n, N;
    uint32_t degree_log, rate_bits, cap_height;
    bool blinding;
    RawVec<u64> coeffs;        // B x n column-major ("polynomials")
    RawVec<u64> leaves;        // N x W row-major
    RawVec<Hash> digests;      // 2*(N-C)
    RawVec<Hash> cap;          // C
};

namespace {
const size_t SALT_SIZE = 4;  // oracle.rs:26

// from_values / from_coeffs / lde_values, oracle.rs:57-139; transpose util/mod.rs:25-31
glo_commit* commit_new(const u64* cols, size_t col_stride, size_t B, uint32_t log_n, uint32_t rate_bits,
                       uint32_t cap_height, const u64* salt, bool is_coeffs, int nthreads) {
    if (cap_height > log_n + rate_bits) {
        fprintf(stderr, "oracle: cap_height=%u should be at most log2(leaves.len())=%u\n", cap_height,
                log_n + rate_bits);  // merkle_tree.rs:195-200
        return nullptr;
    }
    glo_commit* c = new glo_commit();
    size_t n = (size_t)1 << log_n, N = n << rate_bits;
    c->B = B;
    c->n = n;
    c->N = N;
    c->degree_log = log_n;
    c->rate_bits = rate_bits;
    c->cap_height = cap_height;
    c->blinding = salt != nullptr;
    size_t W = B + (salt ? SALT_SIZE : 0);
    c->W = W;
    c->coeffs.resize(B * n);
    // "IFFT": values.into_par_iter().map(|v| v.ifft())   (root table rebuilt per call: fft.rs:41)
    RootTable rt_n = fft_root_table(n);
    parallel_for(B, nthreads, [&](size_t b) {
        u64* dst = c->coeffs.data() + b * n;
        memcpy(dst, cols + b * col_stride, n * 8);
        if (!is_coeffs) ifft_with_options(dst, n, &rt_n);
        else
            for (size_t i = 0; i < n; i++) dst[i] = canon(dst[i]);
    });
    // "FFT + blinding": lde_values
    RootTable rt_N = fft_root_table(N);
    RawVec<u64> lde;  // column-major Vec<Vec<F>>
    lde.resize(W * N);
    parallel_for(B, nthreads, [&](size_t b) {
        u64* src = c->coeffs.data() + b * n;
        for (size_t i = 0; i < n; i++) src[i] = canon(src[i]);
        u64* dst = lde.data() + b * N;
        memcpy(dst, src, n * 8);
        memset(dst + n, 0, (N - n) * 8);  // p.lde(rate_bits): zero-pad
        coset_fft_with_options(dst, N, MULTIPLICATIVE_GROUP_GENERATOR, rate_bits, &rt_N);
    });
    if (salt)
        for (size_t s = 0; s < SALT_SIZE; s++) memcpy(lde.data() + (B + s) * N, salt + s * N, N * 8);
    // "transpose LDEs" + reverse_index_bits_in_place(&mut leaves) (oracle.rs:97-98): the reference transposes
    // into one Vec per LDE point and then permutes the Vec headers; writing row i straight to position
    // bitrev(i) is the same permutation without moving W-word rows twice. Blocks of 8 consecutive LDE points
    // (one cache line of every column) per step, like the reference's blocked transpose (util/mod.rs:25-31).
    c->leaves.resize(N * W);
    const uint32_t lgN = log_n + rate_bits;
    const size_t TB = N >= 8 ? 8 : N;
    parallel_for(N / TB, nthreads, [&](size_t blk) {
        u64* rows[8];
        for (size_t k = 0; k < TB; k++) rows[k] = c->leaves.data() + (size_t)reverse_bits(blk * TB + k, lgN) * W;
        for (size_t b = 0; b < W; b++) {
            const u64* src = lde.data() + b * N + blk * TB;
            for (size_t k = 0; k < TB; k++) rows[k][b] = canon(src[k]);
        }
    }, 64);
    lde.clear();
    // "build Merkle tree"
    size_t C = (size_t)1 << cap_height;
    c->digests.resize(2 * (N - C));
    c->cap.resize(C);
    merkle_build(c->leaves.data(), N, W, cap_height, c->digests.data(), c->cap.data(), nthreads);
    return c;
}
}  // namespace

// ------------------------------------------------------------------ Challenger
struct glo_challenger {
    u64 sponge_state[12];
    std::vector<u64> input_buffer, output_buffer;
};
namespace {
// duplexing, challenger.rs:129-144
void duplexing(glo_challenger* ch) {
    assert(ch->input_buffer.size() <= 8);
    for (size_t i = 0; i < ch->input_buffer.size(); i++) ch->sponge_state[i] = ch->input_buffer[i];
    ch->input_buffer.clear();
    poseidon(ch->sponge_state);
    ch->output_buffer.assign(ch->sponge_state, ch->sponge_state + 8);
}
// observe_element, challenger.rs:39-48
void observe_element(glo_challenger* ch, u64 e) {
    ch->output_buffer.clear();
    ch->input_buffer.push_back(canon(e));
    if (ch->input_buffer.size() == 8) duplexing(ch);
}
void observe_hash(glo_challenger* ch, const Hash& h) {
    for (int i = 0; i < 4; i++) observe_element(ch, h.e[i]);
}
void observe_cap(glo_challenger* ch, const std::vector<Hash>& cap) {
    for (auto& h : cap) observe_hash(ch, h);
}
// get_challenge, challenger.rs:82-92
u64 get_challenge(glo_challenger* ch) {
    if (!ch->input_buffer.empty() || ch->output_buffer.empty()) duplexing(ch);
    u64 v = ch->output_buffer.back();
    ch->output_buffer.pop_back();
    return canon(v);
}
// get_extension_challenge, challenger.rs:109-116
E2 get_extension_challenge(glo_challenger* ch) {
    u64 a = get_challenge(ch);
    u64 b = get_challenge(ch);
    return E2{a, b};
}
void observe_ext(glo_challenger* ch, E2 x) {
    observe_element(ch, x.a);
    observe_element(ch, x.b);
}

// ------------------------------------------------------------------ FRI prover
struct Tree {
    size_t N, W;
    uint32_t cap_height;
    std::vector<u64> leaves;
    std::vector<Hash> digests, cap;
};

void put_u64(std::vector<uint8_t>& out, u64 v) {
    v = canon(v);
    for (int i = 0; i < 8; i++) out.push_back((uint8_t)(v >> (8 * i)));  // write_field: LE canonical
}
void put_hash(std::vector<uint8_t>& out, const Hash& h) {
    for (int i = 0; i < 4; i++) put_u64(out, h.e[i]);
}

// ext polynomial coset FFT: shift and roots are base-field, so it acts per component
// (field/src/field_testing.rs:167-178)
void ext_coset_fft(std::vector<E2>& v, u64 shift) {
    size_t n = v.size();
    std::vector<u64> a(n), b(n);
    for (size_t i = 0; i < n; i++) {
        a[i] = v[i].a;
        b[i] = v[i].b;
    }
    coset_fft_with_options(a.data(), n, shift, 0, nullptr);
    coset_fft_with_options(b.data(), n, shift, 0, nullptr);
    for (size_t i = 0; i < n; i++) v[i] = E2{canon(a[i]), canon(b[i])};
}
void ext_coset_ifft(std::vector<E2>& v, u64 shift) {
    size_t n = v.size();
    std::vector<u64> a(n), b(n);
    for (size_t i = 0; i < n; i++) {
        a[i] = v[i].a;
        b[i] = v[i].b;
    }
    coset_ifft(a.data(), n, shift);
    coset_ifft(b.data(), n, shift);
    for (size_t i = 0; i < n; i++) v[i] = E2{canon(a[i]), canon(b[i])};
}
}  // namespace

// ------------------------------------------------------------------ batch FRI (SURVEY 8f-4)
// BatchFriOracle::from_coeffs (batch_fri/oracle.rs:71-131) + BatchMerkleTree::new (hash/batch_merkle_tree.rs:34-128)
struct glo_batch_commit {
    struct Group {
        uint32_t degree_bits;
        size_t B, n, N;
        std::vector<u64> coeffs;  // B x n
        std::vector<u64> leaves;  // N x B row-major, leaf j = LDE row bitrev(j)
    };
    struct Stage {
        size_t N, W;
        uint32_t cap_height;
        std::vector<u64> rows;    // N x W (stage 0: the group's leaves; later: previous cap digest || group row)
        std::vector<Hash> digests, cap;
    };
    uint32_t rate_bits, cap_height;
    std::vector<Group> groups;
    std::vector<Stage> stages;
    std::vector<std::pair<size_t, size_t>> where;  // polynomial index -> (group, index in group)
};

extern "C" {

uint64_t glo_canon(uint64_t a) { return canon(a); }
uint64_t glo_add(uint64_t a, uint64_t b) { return canon(fadd(a, b)); }
uint64_t glo_sub(uint64_t a, uint64_t b) { return canon(fsub(a, b)); }
uint64_t glo_mul(uint64_t a, uint64_t b) { return canon(fmul(a, b)); }
uint64_t glo_neg(uint64_t a) { return fneg(a); }
uint64_t glo_inv(uint64_t a) { return canon(finv(a)); }
uint64_t glo_exp(uint64_t a, uint64_t e) { return canon(fexp(a, e)); }
uint64_t glo_primitive_root_of_unity(uint32_t k) { return canon(primitive_root_of_unity(k)); }
uint64_t glo_inverse_2exp(uint32_t k) { return canon(inverse_2exp(k)); }
uint64_t glo_coset_shift(void) { return MULTIPLICATIVE_GROUP_GENERATOR; }
void glo_ext2_mul(const uint64_t a[2], const uint64_t b[2], uint64_t out[2]) {
    E2 r = emul(E2{a[0], a[1]}, E2{b[0], b[1]});
    out[0] = canon(r.a);
    out[1] = canon(r.b);
}
void glo_ext2_inv(const uint64_t a[2], uint64_t out[2]) {
    E2 r = einv(E2{a[0], a[1]});
    out[0] = canon(r.a);
    out[1] = canon(r.b);
}

uint64_t glo_reverse_bits(uint64_t x, uint32_t bits) { return reverse_bits(x, bits); }
void glo_reverse_index_bits_in_place(uint64_t* arr, size_t n, size_t w) { reverse_index_bits_in_place(arr, n, w); }

void glo_fft(uint64_t* buf, uint32_t log_n, uint32_t zf) {
    size_t n = (size_t)1 << log_n;
    fft_with_options(buf, n, zf, nullptr);
    for (size_t i = 0; i < n; i++) buf[i] = canon(buf[i]);
}
void glo_ifft(uint64_t* buf, uint32_t log_n) {
    size_t n = (size_t)1 << log_n;
    ifft_with_options(buf, n, nullptr);
    for (size_t i = 0; i < n; i++) buf[i] = canon(buf[i]);
}
void glo_coset_fft(uint64_t* buf, uint32_t log_n, uint64_t shift, uint32_t zf) {
    size_t n = (size_t)1 << log_n;
    coset_fft_with_options(buf, n, shift, zf, nullptr);
    for (size_t i = 0; i < n; i++) buf[i] = canon(buf[i]);
}
void glo_coset_ifft(uint64_t* buf, uint32_t log_n, uint64_t shift) {
    size_t n = (size_t)1 << log_n;
    coset_ifft(buf, n, shift);
    for (size_t i = 0; i < n; i++) buf[i] = canon(buf[i]);
}
// evaluate_naive on the coset, field/src/fft.rs:251-282 / polynomial/mod.rs:476-516
void glo_naive_coset_eval(const uint64_t* coeffs, uint32_t log_n, uint64_t shift, uint64_t* out) {
    size_t n = (size_t)1 << log_n;
    u64 w = primitive_root_of_unity(log_n);
    u64 x = shift;
    for (size_t i = 0; i < n; i++) {
        u64 acc = 0;
        for (size_t k = n; k-- > 0;) acc = fadd(fmul(acc, x), coeffs[k]);
        out[i] = canon(acc);
        x = fmul(x, w);
    }
}

void glo_poseidon(uint64_t st[12]) {
    poseidon(st);
    for (int i = 0; i < 12; i++) st[i] = canon(st[i]);
}
void glo_poseidon_naive(uint64_t st[12]) {
    poseidon_naive(st);
    for (int i = 0; i < 12; i++) st[i] = canon(st[i]);
}
void glo_poseidon_many(uint64_t* states, size_t n, int nthreads) {
    parallel_for(n, std::max(1, nthreads), [&](size_t i) { glo_poseidon(states + 12 * i); }, 1024);
}
uint64_t glo_pow_min_nonce(const uint64_t state[12], uint32_t pos, uint32_t min_leading_zeros, uint64_t limit,
                           int nthreads) {
    // fri_proof_of_work (prover.rs:183-194): the first nonce in increasing order whose permuted lane 7 has enough
    // leading zeros. Candidates go in blocks of increasing order; inside a block the threads keep the smallest hit.
    const size_t GRAIN = 4096;
    const int T = std::max(1, nthreads);
    const u64 block = (u64)GRAIN * T * 4;
    for (u64 start = 0; start < limit; start += block) {
        const u64 count = std::min<u64>(block, limit - start);
        std::atomic<u64> best{~0ULL};
        parallel_for(count, T, [&](size_t i) {
            const u64 cand = start + i;
            if (cand >= best.load(std::memory_order_relaxed)) return;
            u64 st[12];
            memcpy(st, state, sizeof(st));
            st[pos] = cand;
            poseidon(st);
            const u64 resp = canon(st[7]);
            const uint32_t lz = resp == 0 ? 64 : (uint32_t)__builtin_clzll(resp);
            if (lz < min_leading_zeros) return;
            u64 cur = best.load();
            while (cand < cur && !best.compare_exchange_weak(cur, cand)) {
            }
        }, GRAIN);
        if (best.load() != ~0ULL) return best.load();
    }
    return ~0ULL;
}
void glo_hash_no_pad(const uint64_t* in, size_t len, uint64_t out[4]) {
    Hash h = hash_no_pad(in, len);
    memcpy(out, h.e, 32);
}
void glo_hash_or_noop(const uint64_t* in, size_t len, uint64_t out[4]) {
    Hash h = hash_or_noop(in, len);
    memcpy(out, h.e, 32);
}
void glo_two_to_one(const uint64_t l[4], const uint64_t r[4], uint64_t out[4]) {
    Hash a, b;
    memcpy(a.e, l, 32);
    memcpy(b.e, r, 32);
    Hash h = two_to_one(a, b);
    memcpy(out, h.e, 32);
}
void glo_hash_many(const uint64_t* in, size_t n_items, size_t W, uint64_t* out, int nthreads) {
    int T = std::max(1, nthreads);
    std::vector<std::thread> ths;
    for (int t = 0; t < T; t++)
        ths.emplace_back([=] {
            size_t lo = n_items * t / T, hi = n_items * (t + 1) / T;
            for (size_t i = lo; i < hi; i++) {
                Hash h = hash_or_noop(in + i * W, W);
                memcpy(out + 4 * i, h.e, 32);
            }
        });
    for (auto& t : ths) t.join();
}

int glo_merkle_build(const uint64_t* leaves, size_t N, size_t W, uint32_t cap_height, uint64_t* digests,
                     uint64_t* cap, int nthreads) {
    return merkle_build(leaves, N, W, cap_height, (Hash*)digests, (Hash*)cap, nthreads);
}
void glo_merkle_prove(size_t leaf_index, size_t N, uint32_t cap_height, const uint64_t* digests,
                      uint64_t* siblings) {
    merkle_prove(leaf_index, N, cap_height, (const Hash*)digests, (Hash*)siblings);
}
int glo_merkle_verify(const uint64_t* leaf, size_t W, size_t leaf_index, const uint64_t* siblings,
                      size_t n_siblings, const uint64_t* cap, uint32_t cap_height) {
    (void)cap_height;
    return merkle_verify(leaf, W, leaf_index, (const Hash*)siblings, n_siblings, (const Hash*)cap) ? 1 : 0;
}

glo_commit* glo_commit_new(const uint64_t* cols, size_t col_stride, size_t B, uint32_t log_n,
                           uint32_t rate_bits, uint32_t cap_height, const uint64_t* salt, int is_coeffs,
                           int nthreads) {
    return commit_new(cols, col_stride, B, log_n, rate_bits, cap_height, salt, is_coeffs != 0, nthreads);
}
void glo_commit_free(glo_commit* c) { delete c; }
size_t glo_commit_leaf_width(const glo_commit* c) { return c->W; }
const uint64_t* glo_commit_coeffs(const glo_commit* c) { return c->coeffs.data(); }
const uint64_t* glo_commit_leaves(const glo_commit* c) { return c->leaves.data(); }
const uint64_t* glo_commit_digests(const glo_commit* c) { return (const u64*)c->digests.data(); }
const uint64_t* glo_commit_cap(const glo_commit* c) { return (const u64*)c->cap.data(); }
// get_lde_values, oracle.rs:142-147
void glo_commit_get_lde_values(const glo_commit* c, size_t index, size_t step, uint64_t* out) {
    size_t idx = reverse_bits(index * step, c->degree_log + c->rate_bits);
    memcpy(out, c->leaves.data() + idx * c->W, c->B * 8);
}

glo_challenger* glo_challenger_new(void) {
    glo_challenger* ch = new glo_challenger();
    memset(ch->sponge_state, 0, sizeof(ch->sponge_state));
    return ch;
}
glo_challenger* glo_challenger_clone(const glo_challenger* c) { return new glo_challenger(*c); }
void glo_challenger_free(glo_challenger* c) { delete c; }
void glo_challenger_observe(glo_challenger* c, const uint64_t* e, size_t n) {
    for (size_t i = 0; i < n; i++) observe_element(c, e[i]);
}
uint64_t glo_challenger_get_challenge(glo_challenger* c) { return get_challenge(c); }
size_t glo_challenger_state(const glo_challenger* c, uint64_t state[12], uint64_t inbuf[8]) {
    for (int i = 0; i < 12; i++) state[i] = canon(c->sponge_state[i]);
    for (size_t i = 0; i < c->input_buffer.size(); i++) inbuf[i] = c->input_buffer[i];
    return c->input_buffer.size();
}

void glo_free(void* p) { free(p); }

// wires_permutation_partial_products_and_zs, plonk/prover.rs:387-449
int glo_partial_products_and_zs(const uint64_t* wires, const uint64_t* sigmas, const uint64_t* k_is, uint32_t log_n,
                                uint32_t num_routed, uint64_t beta, uint64_t gamma, uint32_t degree, uint64_t* out) {
    const size_t n = (size_t)1 << log_n;
    const size_t num_chunks = (num_routed + degree - 1) / degree;  // quotient_chunk_products length
    const size_t num_prods = num_chunks - 1;                        // num_partial_products, partial_products.rs:40-47
    // subgroup = two_adic_subgroup(degree_bits)
    const u64 w = primitive_root_of_unity(log_n);
    u64 x = 1, z_x = 1;
    std::vector<u64> q(num_routed), chunkp(num_chunks);
    for (size_t i = 0; i < n; i++) {
        for (uint32_t j = 0; j < num_routed; j++) {
            u64 wire = wires[(size_t)j * n + i];
            u64 num = fadd(fadd(wire, fmul(beta, fmul(k_is[j], x))), gamma);
            u64 den = fadd(fadd(wire, fmul(beta, sigmas[(size_t)j * n + i])), gamma);
            if (canon(den) == 0) return 1;
            q[j] = fmul(num, finv(den));
        }
        // quotient_chunk_products, partial_products.rs:13-24
        for (size_t m = 0; m < num_chunks; m++) {
            u64 p = 1;
            for (size_t j = m * degree; j < std::min<size_t>((m + 1) * degree, num_routed); j++) p = fmul(p, q[j]);
            chunkp[m] = p;
        }
        // partial_products_and_z_gx, partial_products.rs:28-37, then swap(z_x, last)
        u64 acc = z_x;
        for (size_t m = 0; m < num_chunks; m++) {
            acc = fmul(acc, chunkp[m]);
            if (m < num_prods) out[m * n + i] = canon(acc);
        }
        out[num_prods * n + i] = canon(z_x);  // the last slot holds Z(x), not Z(gx)
        z_x = acc;
        x = fmul(x, w);
    }
    return 0;
}

// ------------------------------------------------------------------ lookup helper polynomials (SURVEY 8f-3)
// compute_lookup_polys, plonky2/src/plonk/prover.rs:458-577, line by line. witness.get_wire(row, w) = wires[w*n + row].
int glo_lookup_polys(const uint64_t* wires, uint32_t log_n, uint32_t num_routed_wires,
                     uint32_t max_quotient_degree_factor, const uint64_t deltas[4], const uint32_t* lookup_rows,
                     uint32_t n_lookup_wires, uint64_t* out) {
    const size_t degree = (size_t)1 << log_n;
    const size_t num_lu_slots = num_routed_wires / 2;         // LookupGate::num_slots, gates/lookup.rs:58-61
    const size_t max_lookup_degree = max_quotient_degree_factor - 1;
    const size_t num_partial_lookups = (num_lu_slots + max_lookup_degree - 1) / max_lookup_degree;
    const size_t num_lut_slots = num_routed_wires / 3;        // LookupTableGate::num_slots, gates/lookup_table.rs:64-67
    const size_t max_lookup_table_degree = (num_lut_slots + num_partial_lookups - 1) / num_partial_lookups;
    auto get_wire = [&](size_t row, size_t w) { return wires[w * degree + row]; };
    auto poly = [&](size_t k) { return out + k * degree; };   // final_poly_vecs[k].values
    for (size_t i = 0; i < (num_partial_lookups + 1) * degree; i++) out[i] = 0;
    const u64 dA = deltas[0], dB = deltas[1], dAlpha = deltas[2], dDelta = deltas[3];
    for (uint32_t lw = 0; lw < n_lookup_wires; lw++) {
        const size_t last_lu_row = lookup_rows[3 * lw], last_lut_row = lookup_rows[3 * lw + 1], first_lut_row = lookup_rows[3 * lw + 2];
        // Set values for partial Sums and RE.
        for (size_t row = first_lut_row + 1; row-- > last_lut_row;) {
            std::vector<u64> looked_combo_inverses(num_lut_slots), lookup_combos(num_lut_slots);
            for (size_t s = 0; s < num_lut_slots; s++) {
                const u64 looked_inp = get_wire(row, 3 * s), looked_out = get_wire(row, 3 * s + 1);
                const u64 minus = fsub(dAlpha, fadd(looked_inp, fmul(dA, looked_out)));
                if (canon(minus) == 0) return 1;  // batch_multiplicative_inverse would panic
                looked_combo_inverses[s] = finv(minus);
                lookup_combos[s] = fadd(looked_inp, fmul(dB, looked_out));
            }
            u64 new_re = poly(0)[row + 1];
            for (u64 elt : lookup_combos) new_re = fadd(fmul(new_re, dDelta), elt);
            poly(0)[row] = canon(new_re);
            for (size_t slot = 0; slot < num_partial_lookups; slot++) {
                u64 sum = slot != 0 ? poly(slot)[row] : poly(num_partial_lookups)[row + 1];
                for (size_t s = slot * max_lookup_table_degree; s < std::min((slot + 1) * max_lookup_table_degree, num_lut_slots); s++)
                    sum = fadd(sum, fmul(get_wire(row, 3 * s + 2), looked_combo_inverses[s]));
                poly(slot + 1)[row] = canon(sum);
            }
        }
        // Set values for partial LDCs.
        for (size_t row = last_lut_row; row-- > last_lu_row;) {
            std::vector<u64> looking_combo_inverses(num_lu_slots);
            for (size_t s = 0; s < num_lu_slots; s++) {
                const u64 looking_in = get_wire(row, 2 * s), looking_out = get_wire(row, 2 * s + 1);
                const u64 minus = fsub(dAlpha, fadd(looking_in, fmul(dA, looking_out)));
                if (canon(minus) == 0) return 1;
                looking_combo_inverses[s] = finv(minus);
            }
            for (size_t slot = 0; slot < num_partial_lookups; slot++) {
                const u64 prev = slot == 0 ? poly(num_partial_lookups)[row + 1] : poly(slot)[row];
                u64 sum = 0;
                for (size_t s = slot * max_lookup_degree; s < std::min((slot + 1) * max_lookup_degree, num_lu_slots); s++)
                    sum = fadd(sum, looking_combo_inverses[s]);
                poly(slot + 1)[row] = canon(fsub(prev, sum));
            }
        }
    }
    return 0;
}

// ------------------------------------------------------------------ STARK quotient (SURVEY 8f-1)
// compute_quotient_polys (starky/src/prover.rs:488-668) for FibonacciStark (starky/src/fibonacci_stark.rs:73-95),
// restated with the reference's own steps: Lagrange selectors by `PolynomialValues::selector(..).lde_onto_coset`
// (ifft, zero-pad, coset FFT), ZeroPolyOnCoset (field/src/zero_poly_coset.rs), the ConstraintConsumer accumulation
// (constraint_consumer.rs:60-84), division by Z_H, transpose, coset_ifft. P::WIDTH = 1 (scalar packing).
int glo_stark_quotient_fibonacci(const glo_commit* trace, const uint64_t pi[3], const uint64_t* alphas,
                                 size_t n_alphas, uint64_t* out) {
    if (trace->B != 2) return 1;
    const uint32_t degree_bits = trace->degree_log, rate_bits = trace->rate_bits;
    const size_t degree = (size_t)1 << degree_bits;
    const size_t constraint_degree = 2;
    const size_t quotient_degree_factor = std::max<size_t>(1, constraint_degree - 1);  // stark.rs:87-92
    uint32_t quotient_degree_bits = 0;
    while (((size_t)1 << quotient_degree_bits) < quotient_degree_factor) quotient_degree_bits++;
    if (quotient_degree_bits > rate_bits) return 2;
    const size_t step = (size_t)1 << (rate_bits - quotient_degree_bits);
    const size_t next_step = (size_t)1 << quotient_degree_bits;
    const size_t size = degree << quotient_degree_bits;
    auto lde_onto_coset = [&](size_t index) {  // selector(degree, index).lde_onto_coset(quotient_degree_bits)
        std::vector<u64> v(size, 0);
        v[index] = 1;
        ifft_with_options(v.data(), degree, nullptr);
        coset_fft_with_options(v.data(), size, MULTIPLICATIVE_GROUP_GENERATOR, quotient_degree_bits, nullptr);
        return v;
    };
    std::vector<u64> lagrange_first = lde_onto_coset(0), lagrange_last = lde_onto_coset(degree - 1);
    // ZeroPolyOnCoset::new(degree_bits, quotient_degree_bits)
    u64 g_pow_n = MULTIPLICATIVE_GROUP_GENERATOR;
    for (uint32_t k = 0; k < degree_bits; k++) g_pow_n = fsqr(g_pow_n);
    const size_t rate = (size_t)1 << quotient_degree_bits;
    std::vector<u64> zh_inv(rate);
    {
        u64 w = primitive_root_of_unity(quotient_degree_bits), x = 1;
        for (size_t j = 0; j < rate; j++) {
            zh_inv[j] = finv(fsub(fmul(g_pow_n, x), 1));
            x = fmul(x, w);
        }
    }
    const u64 last = finv(primitive_root_of_unity(degree_bits));
    const u64 wsize = primitive_root_of_unity(degree_bits + quotient_degree_bits);
    std::vector<u64> coset(size);
    {
        u64 x = MULTIPLICATIVE_GROUP_GENERATOR;  // cyclic_subgroup_coset_known_order(w, shift, size)
        for (size_t i = 0; i < size; i++) {
            coset[i] = x;
            x = fmul(x, wsize);
        }
    }
    std::vector<u64> quotient_values(size * n_alphas);  // [i][j]
    u64 lv[2], nv[2];
    for (size_t i_start = 0; i_start < size; i_start++) {
        const size_t i_next_start = (i_start + next_step) % size;
        const u64 x = coset[i_start];
        const u64 z_last = fsub(x, last);
        glo_commit_get_lde_values(trace, i_start, step, lv);
        glo_commit_get_lde_values(trace, i_next_start, step, nv);
        std::vector<u64> acc(n_alphas, 0);
        auto constraint = [&](u64 c) {
            for (size_t j = 0; j < n_alphas; j++) acc[j] = fadd(fmul(acc[j], alphas[j]), c);
        };
        // eval_packed_generic, fibonacci_stark.rs:73-95
        constraint(fmul(fsub(lv[0], pi[0]), lagrange_first[i_start]));
        constraint(fmul(fsub(lv[1], pi[1]), lagrange_first[i_start]));
        constraint(fmul(fsub(lv[1], pi[2]), lagrange_last[i_start]));
        constraint(fmul(fsub(nv[0], lv[1]), z_last));
        constraint(fmul(fsub(fsub(nv[1], lv[0]), lv[1]), z_last));
        const u64 denominator_inv = zh_inv[i_start % rate];
        for (size_t j = 0; j < n_alphas; j++) quotient_values[i_start * n_alphas + j] = fmul(acc[j], denominator_inv);
    }
    for (size_t j = 0; j < n_alphas; j++) {  // transpose + coset_ifft
        u64* col = out + j * size;
        for (size_t i = 0; i < size; i++) col[i] = quotient_values[i * n_alphas + j];
        coset_ifft(col, size, MULTIPLICATIVE_GROUP_GENERATOR);
        for (size_t i = 0; i < size; i++) col[i] = canon(col[i]);
    }
    return 0;
}

// compute_quotient_polys (plonky2/src/plonk/prover.rs:609-815) with eval_vanishing_poly_base_batch
// (plonk/vanishing_poly.rs:167-340, no lookups) for circuits made of NoopGate, ConstantGate, PublicInputGate and
// ArithmeticGate (gates/{noop,constant,public_input,arithmetic_base}.rs), restated with the reference's own steps:
// evaluate_gate_constraints_base_batch (vanishing_poly.rs:702-728) with compute_filter (gates/gate.rs:326-333),
// L_0(x)(Z(x) - 1), check_partial_products (util/partial_products.rs:52-76), reduce_with_powers_multi
// (plonk_common.rs:99-116), ZeroPolyOnCoset (field/src/zero_poly_coset.rs), transpose, coset_ifft. BATCH_SIZE = 1.
static const u64 UNUSED_SELECTOR = 0xFFFFFFFFull;  // gates/selectors.rs:14
static void gate_eval_unfiltered(const glo_gate& g, const u64* local_constants, const u64* local_wires,
                                 const uint64_t public_inputs_hash[4], std::vector<u64>& res) {
    res.clear();
    switch (g.kind) {
        case GLO_GATE_NOOP: break;
        case GLO_GATE_CONSTANT:  // constant.rs:121-129
            for (uint32_t i = 0; i < g.param; i++) res.push_back(fsub(local_constants[i], local_wires[i]));
            break;
        case GLO_GATE_PUBLIC_INPUT:  // public_input.rs:103-113
            for (uint32_t i = 0; i < 4; i++) res.push_back(fsub(local_wires[i], public_inputs_hash[i]));
            break;
        case GLO_GATE_ARITHMETIC: {  // arithmetic_base.rs:168-185
            const u64 const_0 = local_constants[0], const_1 = local_constants[1];
            for (uint32_t i = 0; i < g.param; i++) {
                const u64 multiplicand_0 = local_wires[4 * i], multiplicand_1 = local_wires[4 * i + 1];
                const u64 addend = local_wires[4 * i + 2], output = local_wires[4 * i + 3];
                const u64 computed_output = fadd(fmul(fmul(multiplicand_0, multiplicand_1), const_0), fmul(addend, const_1));
                res.push_back(fsub(output, computed_output));
            }
            break;
        }
        case GLO_GATE_ARITHMETIC_EXTENSION: {  // arithmetic_extension.rs:92-110
            const u64 const_0 = local_constants[0], const_1 = local_constants[1];
            auto ext = [&](size_t at) { return E2{local_wires[at], local_wires[at + 1]}; };
            for (uint32_t i = 0; i < g.param; i++) {
                const E2 multiplicand_0 = ext(8 * i), multiplicand_1 = ext(8 * i + 2), addend = ext(8 * i + 4), output = ext(8 * i + 6);
                const E2 computed_output = eadd(escale(emul(multiplicand_0, multiplicand_1), const_0), escale(addend, const_1));
                const E2 d = esub(output, computed_output);
                res.push_back(d.a);
                res.push_back(d.b);
            }
            break;
        }
        case GLO_GATE_MUL_EXTENSION: {  // multiplication_extension.rs:86-101
            const u64 const_0 = local_constants[0];
            auto ext = [&](size_t at) { return E2{local_wires[at], local_wires[at + 1]}; };
            for (uint32_t i = 0; i < g.param; i++) {
                const E2 d = esub(ext(6 * i + 4), escale(emul(ext(6 * i), ext(6 * i + 2)), const_0));
                res.push_back(d.a);
                res.push_back(d.b);
            }
            break;
        }
        case GLO_GATE_BASE_SUM: {  // base_sum.rs:153-170, BaseSumGate<B = param2> with param limbs
            const u64 B = g.param2, sum = local_wires[0];
            const u64* limbs = local_wires + 1;
            u64 computed_sum = 0;  // reduce_with_powers(limbs, B), plonk_common.rs:128-135
            for (size_t i = g.param; i-- > 0;) computed_sum = fadd(fmul(computed_sum, B), limbs[i]);
            res.push_back(fsub(computed_sum, sum));
            for (uint32_t l = 0; l < g.param; l++) {
                u64 prod = 1;
                for (u64 i = 0; i < B; i++) prod = fmul(prod, fsub(limbs[l], i));
                res.push_back(prod);
            }
            break;
        }
        case GLO_GATE_REDUCING: case GLO_GATE_REDUCING_EXTENSION: {  // reducing.rs:107-127, reducing_extension.rs:109-128
            const bool ext_coeffs = g.kind == GLO_GATE_REDUCING_EXTENSION;
            const size_t num_coeffs = g.param, start_coeffs = 6;
            const size_t start_accs = start_coeffs + num_coeffs * (ext_coeffs ? 2 : 1);
            auto ext = [&](size_t at) { return E2{local_wires[at], local_wires[at + 1]}; };
            const E2 alpha = ext(2), old_acc = ext(4);
            E2 acc = old_acc;
            for (size_t i = 0; i < num_coeffs; i++) {
                const E2 coeff = ext_coeffs ? ext(start_coeffs + 2 * i) : e2(local_wires[start_coeffs + i]);
                const E2 acc_i = ext(i == num_coeffs - 1 ? 0 : start_accs + 2 * i);  // the last accumulator is the output
                const E2 d = esub(eadd(emul(acc, alpha), coeff), acc_i);
                res.push_back(d.a);
                res.push_back(d.b);
                acc = acc_i;
            }
            break;
        }
        case GLO_GATE_POSEIDON_MDS: {  // poseidon_mds.rs:156-175, mds_layer_field (hash/poseidon.rs:292-306) per component
            u64 in_a[12], in_b[12];
            for (int i = 0; i < 12; i++) {
                in_a[i] = local_wires[2 * i];
                in_b[i] = local_wires[2 * i + 1];
            }
            mds_layer(in_a);
            mds_layer(in_b);
            for (int i = 0; i < 12; i++) {
                res.push_back(fsub(local_wires[2 * (12 + i)], in_a[i]));
                res.push_back(fsub(local_wires[2 * (12 + i) + 1], in_b[i]));
            }
            break;
        }
        case GLO_GATE_RANDOM_ACCESS: {  // random_access.rs:302-343; param = bits, param2 = num_copies, param3 = extra constants
            const size_t bits = g.param, num_copies = g.param2, num_extra = g.param3, vec_size = (size_t)1 << bits;
            const size_t num_routed = (2 + vec_size) * num_copies + num_extra;
            for (size_t copy = 0; copy < num_copies; copy++) {
                const u64 access_index = local_wires[(2 + vec_size) * copy];
                const u64 claimed_element = local_wires[(2 + vec_size) * copy + 1];
                std::vector<u64> list_items(local_wires + (2 + vec_size) * copy + 2, local_wires + (2 + vec_size) * (copy + 1));
                const u64* b = local_wires + num_routed + copy * bits;
                for (size_t i = 0; i < bits; i++) res.push_back(fmul(b[i], fsub(b[i], 1)));
                u64 reconstructed_index = 0;
                for (size_t i = bits; i-- > 0;) reconstructed_index = fadd(fadd(reconstructed_index, reconstructed_index), b[i]);
                res.push_back(fsub(reconstructed_index, access_index));
                for (size_t i = 0; i < bits; i++) {
                    std::vector<u64> next(list_items.size() / 2);
                    for (size_t k = 0; k < next.size(); k++) {
                        const u64 x = list_items[2 * k], y = list_items[2 * k + 1];
                        next[k] = fadd(x, fmul(b[i], fsub(y, x)));
                    }
                    list_items.swap(next);
                }
                res.push_back(fsub(list_items[0], claimed_element));
            }
            for (size_t i = 0; i < num_extra; i++) res.push_back(fsub(local_constants[i], local_wires[(2 + vec_size) * num_copies + i]));
            break;
        }
        case GLO_GATE_EXPONENTIATION: {  // exponentiation.rs:210-243; param = num_power_bits
            const size_t n = g.param;
            const u64 base = local_wires[0], output = local_wires[1 + n];
            const u64* power_bits = local_wires + 1;
            const u64* intermediate_values = local_wires + 2 + n;
            for (size_t i = 0; i < n; i++) {
                const u64 prev_intermediate_value = i == 0 ? 1 : fsqr(intermediate_values[i - 1]);
                const u64 cur_bit = power_bits[n - i - 1];
                const u64 not_cur_bit = fsub(1, cur_bit);
                const u64 computed_intermediate_value = fmul(prev_intermediate_value, fadd(fmul(cur_bit, base), not_cur_bit));
                res.push_back(fsub(computed_intermediate_value, intermediate_values[i]));
            }
            res.push_back(fsub(output, intermediate_values[n - 1]));
            break;
        }
        case GLO_GATE_COSET_INTERPOLATION: {  // coset_interpolation.rs:251-298,553-580; param = subgroup_bits, param2 = degree
            const size_t num_points = (size_t)1 << g.param, degree = g.param2;
            const size_t num_intermediates = (num_points - 2) / (degree - 1);
            const size_t start_evaluation_point = 1 + 2 * num_points, start_evaluation_value = start_evaluation_point + 2;
            const size_t start_intermediates = start_evaluation_value + 2;
            auto ext = [&](size_t at) { return E2{local_wires[at], local_wires[at + 1]}; };
            std::vector<u64> domain(num_points), weights(num_points);  // two_adic_subgroup, barycentric_weights (interpolation.rs:53-65)
            {
                const u64 w = primitive_root_of_unity((uint32_t)g.param);
                u64 x = 1;
                for (size_t i = 0; i < num_points; i++, x = fmul(x, w)) domain[i] = x;
                for (size_t i = 0; i < num_points; i++) {
                    u64 d = 1;
                    for (size_t j = 0; j < num_points; j++)
                        if (j != i) d = fmul(d, fsub(domain[i], domain[j]));
                    weights[i] = finv(d);
                }
            }
            const u64 shift = local_wires[0];
            const E2 evaluation_point = ext(start_evaluation_point);
            const E2 shifted_evaluation_point = ext(start_intermediates + 2 * 2 * num_intermediates);
            {
                const E2 d = esub(evaluation_point, escale(shifted_evaluation_point, shift));
                res.push_back(d.a);
                res.push_back(d.b);
            }
            auto partial_interpolate = [&](size_t lo, size_t hi, E2& eval, E2& terms_partial_prod) {
                for (size_t i = lo; i < hi; i++) {
                    const E2 val = escale(ext(1 + 2 * i), weights[i]);
                    const E2 term = esub(shifted_evaluation_point, e2(domain[i]));
                    const E2 next_eval = eadd(emul(eval, term), emul(val, terms_partial_prod));
                    terms_partial_prod = emul(terms_partial_prod, term);
                    eval = next_eval;
                }
            };
            E2 computed_eval = e2(0), computed_prod = e2(1);
            partial_interpolate(0, degree, computed_eval, computed_prod);
            for (size_t i = 0; i < num_intermediates; i++) {
                const E2 intermediate_eval = ext(start_intermediates + 2 * i);
                const E2 intermediate_prod = ext(start_intermediates + 2 * (num_intermediates + i));
                const E2 d0 = esub(intermediate_eval, computed_eval), d1 = esub(intermediate_prod, computed_prod);
                res.push_back(d0.a);
                res.push_back(d0.b);
                res.push_back(d1.a);
                res.push_back(d1.b);
                const size_t start_index = 1 + (degree - 1) * (i + 1);
                const size_t end_index = std::min(start_index + degree - 1, num_points);
                computed_eval = intermediate_eval;
                computed_prod = intermediate_prod;
                partial_interpolate(start_index, end_index, computed_eval, computed_prod);
            }
            const E2 d = esub(ext(start_evaluation_value), computed_eval);
            res.push_back(d.a);
            res.push_back(d.b);
            break;
        }
        case GLO_GATE_POSEIDON: {  // poseidon.rs:204-283 (wire layout :43-101), with the layers of hash/poseidon.rs
            const int W = 12, HALF = GL_POSEIDON_HALF_FULL_ROUNDS, NP = GL_POSEIDON_PARTIAL_ROUNDS;
            const int WIRE_SWAP = 2 * W, START_DELTA = 2 * W + 1, START_FULL_0 = START_DELTA + 4;
            const int START_PARTIAL = START_FULL_0 + W * (HALF - 1), START_FULL_1 = START_PARTIAL + NP;
            const u64 swap = local_wires[WIRE_SWAP];
            res.push_back(fmul(swap, fsub(swap, 1)));
            for (int i = 0; i < 4; i++)
                res.push_back(fsub(fmul(swap, fsub(local_wires[i + 4], local_wires[i])), local_wires[START_DELTA + i]));
            u64 state[12];
            for (int i = 0; i < 4; i++) {
                const u64 delta_i = local_wires[START_DELTA + i];
                state[i] = fadd(local_wires[i], delta_i);
                state[i + 4] = fsub(local_wires[i + 4], delta_i);
            }
            for (int i = 8; i < W; i++) state[i] = local_wires[i];
            int round_ctr = 0;
            for (int r = 0; r < HALF; r++) {
                constant_layer(state, round_ctr);
                if (r != 0)
                    for (int i = 0; i < W; i++) {
                        const u64 sbox_in = local_wires[START_FULL_0 + W * (r - 1) + i];
                        res.push_back(fsub(state[i], sbox_in));
                        state[i] = sbox_in;
                    }
                for (int i = 0; i < W; i++) state[i] = sbox(state[i]);
                mds_layer(state);
                round_ctr++;
            }
            for (int i = 0; i < W; i++) state[i] = fadd(state[i], GL_POSEIDON_FAST_FIRST_RC[i]);
            mds_partial_layer_init(state);
            for (int r = 0; r < NP; r++) {
                const u64 sbox_in = local_wires[START_PARTIAL + r];
                res.push_back(fsub(state[0], sbox_in));
                state[0] = sbox(sbox_in);
                if (r < NP - 1) state[0] = fadd(state[0], GL_POSEIDON_FAST_RC[r]);
                mds_partial_layer_fast(state, r);
            }
            round_ctr += NP;
            for (int r = 0; r < HALF; r++) {
                constant_layer(state, round_ctr);
                for (int i = 0; i < W; i++) {
                    const u64 sbox_in = local_wires[START_FULL_1 + W * r + i];
                    res.push_back(fsub(state[i], sbox_in));
                    state[i] = sbox_in;
                }
                for (int i = 0; i < W; i++) state[i] = sbox(state[i]);
                mds_layer(state);
                round_ctr++;
            }
            for (int i = 0; i < W; i++) res.push_back(fsub(state[i], local_wires[W + i]));
            break;
        }
    }
}

// check_lookup_constraints_batch (plonk/vanishing_poly.rs:521-689) for one challenge
static void check_lookup_constraints_batch(const glo_circuit* cd, const u64* local_wires, const u64* local_lookup_zs,
                                           const u64* next_lookup_zs, const u64* lookup_selectors, const uint64_t deltas[4],
                                           const std::vector<u64>& lut_re_poly_evals, std::vector<u64>& constraints) {
    const size_t num_lu_slots = cd->num_routed_wires / 2, num_lut_slots = cd->num_routed_wires / 3;
    const size_t lu_degree = cd->quotient_degree_factor - 1;
    const size_t num_sldc_polys = cd->num_lookup_polys - 1;
    const size_t lut_degree = (num_lut_slots + num_sldc_polys - 1) / num_sldc_polys;
    const u64 z_re = local_lookup_zs[0], next_z_re = next_lookup_zs[0];
    const u64* z_x_lookup_sldcs = local_lookup_zs + 1;
    const u64* z_gx_lookup_sldcs = next_lookup_zs + 1;
    const u64 delta_a = deltas[0], delta_b = deltas[1], delta_alpha = deltas[2], delta_delta = deltas[3];
    std::vector<u64> current_looked_combos(num_lut_slots), current_looking_combos(num_lu_slots), current_lookup_combos(num_lut_slots);
    for (size_t s = 0; s < num_lut_slots; s++) {
        current_looked_combos[s] = fadd(local_wires[3 * s], fmul(delta_a, local_wires[3 * s + 1]));
        current_lookup_combos[s] = fadd(local_wires[3 * s], fmul(delta_b, local_wires[3 * s + 1]));
    }
    for (size_t s = 0; s < num_lu_slots; s++) current_looking_combos[s] = fadd(local_wires[2 * s], fmul(delta_a, local_wires[2 * s + 1]));
    const size_t TransSre = 0, TransLdc = 1, InitSre = 2, LastLdc = 3, StartEnd = 4;  // LookupSelectors, gates/selectors.rs:33-40
    constraints.push_back(fmul(lookup_selectors[LastLdc], z_x_lookup_sldcs[num_sldc_polys - 1]));
    constraints.push_back(fmul(lookup_selectors[InitSre], z_x_lookup_sldcs[0]));
    constraints.push_back(fmul(lookup_selectors[InitSre], z_re));
    for (size_t r = StartEnd; r < cd->num_lookup_selectors; r++)
        constraints.push_back(fmul(lookup_selectors[r], fsub(z_re, lut_re_poly_evals[r - StartEnd])));
    u64 cur_sum = next_z_re;
    for (u64 elt : current_lookup_combos) cur_sum = fadd(fmul(cur_sum, delta_delta), elt);
    constraints.push_back(fmul(lookup_selectors[TransSre], fsub(z_re, cur_sum)));
    for (size_t poly = 0; poly < num_sldc_polys; poly++) {
        const size_t lut_lo = poly * lut_degree, lut_hi = std::min((poly + 1) * lut_degree, num_lut_slots);
        const size_t lu_lo = poly * lu_degree, lu_hi = std::min((poly + 1) * lu_degree, num_lu_slots);
        u64 lut_prod = 1, lu_prod = 1;
        for (size_t i = lut_lo; i < lut_hi; i++) lut_prod = fmul(lut_prod, fsub(delta_alpha, current_looked_combos[i]));
        for (size_t i = lu_lo; i < lu_hi; i++) lu_prod = fmul(lu_prod, fsub(delta_alpha, current_looking_combos[i]));
        auto lut_prod_i = [&](size_t i) {
            u64 p = 1;
            for (size_t j = lut_lo; j < lut_hi; j++)
                if (j != i) p = fmul(p, fsub(delta_alpha, current_looked_combos[j]));
            return p;
        };
        auto lu_prod_i = [&](size_t i) {
            u64 p = 1;
            for (size_t j = lu_lo; j < lu_hi; j++)
                if (j != i) p = fmul(p, fsub(delta_alpha, current_looking_combos[j]));
            return p;
        };
        u64 lu_sum_prods = 0, lut_sum_prods_with_mul = 0;
        for (size_t i = lu_lo; i < lu_hi; i++) lu_sum_prods = fadd(lu_sum_prods, lu_prod_i(i));
        for (size_t i = lut_lo; i < lut_hi; i++)
            lut_sum_prods_with_mul = fadd(lut_sum_prods_with_mul, fmul(local_wires[3 * i + 2], lut_prod_i(i)));
        const u64 prev = poly == 0 ? z_gx_lookup_sldcs[num_sldc_polys - 1] : z_x_lookup_sldcs[poly - 1];
        const u64 unfiltered_sum_transition = fsub(fmul(lut_prod, fsub(z_x_lookup_sldcs[poly], prev)), lut_sum_prods_with_mul);
        constraints.push_back(fmul(lookup_selectors[TransSre], unfiltered_sum_transition));
        const u64 unfiltered_ldc_transition = fadd(fmul(lu_prod, fsub(z_x_lookup_sldcs[poly], prev)), lu_sum_prods);
        constraints.push_back(fmul(lookup_selectors[TransLdc], unfiltered_ldc_transition));
    }
}

int glo_plonk_quotient(const glo_circuit* cd, const glo_commit* constants_sigmas, const glo_commit* wires,
                       const glo_commit* zs_partial_products, const uint64_t public_inputs_hash[4], const uint64_t* betas,
                       const uint64_t* gammas, const uint64_t* deltas, const uint64_t* alphas, uint64_t* out) {
    const bool has_lookup = cd->num_lookup_polys != 0;
    const uint32_t degree_bits = wires->degree_log, rate_bits = wires->rate_bits;
    if (constants_sigmas->degree_log != degree_bits || zs_partial_products->degree_log != degree_bits) return 1;
    if (constants_sigmas->rate_bits != rate_bits || zs_partial_products->rate_bits != rate_bits) return 1;
    const size_t num_challenges = cd->num_challenges, num_routed_wires = cd->num_routed_wires;
    const size_t num_prods = cd->num_partial_products, max_degree = cd->quotient_degree_factor;
    if (constants_sigmas->B != cd->num_constants + num_routed_wires || wires->B != cd->num_wires ||
        zs_partial_products->B != num_challenges * (1 + num_prods + cd->num_lookup_polys))
        return 3;
    // lut_re_poly_evals (prover.rs:653-681): get_lut_poly(..).eval(delta) (vanishing_poly.rs:30-52) per challenge and table
    std::vector<std::vector<u64>> lut_re_poly_evals(num_challenges);
    if (has_lookup) {
        const size_t nb_slots = num_routed_wires / 3;
        for (size_t c = 0; c < num_challenges; c++) {
            const u64 b = deltas[4 * c + 1], delta = deltas[4 * c + 3];
            size_t at = 0;
            for (size_t t = 0; t < cd->n_luts; t++) {
                const size_t n = cd->lut_len[t];
                const size_t nb_padded_elts = (nb_slots - n % nb_slots) % nb_slots;
                std::vector<u64> coeffs;
                for (size_t k = 0; k < n; k++) coeffs.push_back(fadd(cd->lut_inp[at + k], fmul(b, cd->lut_out[at + k])));
                for (size_t k = 0; k < nb_padded_elts; k++) coeffs.push_back(fadd(cd->lut_inp[at], fmul(b, cd->lut_out[at])));
                std::reverse(coeffs.begin(), coeffs.end());  // degree = n + padding: no zero coefficients to append
                u64 acc = 0;                                 // PolynomialCoeffs::eval: Horner from the top coefficient
                for (size_t k = coeffs.size(); k-- > 0;) acc = fadd(fmul(acc, delta), coeffs[k]);
                lut_re_poly_evals[c].push_back(acc);
                at += n;
            }
        }
    }
    if (num_prods + 1 != (num_routed_wires + max_degree - 1) / max_degree) return 4;  // num_partial_products, partial_products.rs:40-46
    uint32_t quotient_degree_bits = 0;
    while (((size_t)1 << quotient_degree_bits) < cd->quotient_degree_factor) quotient_degree_bits++;
    if (quotient_degree_bits > rate_bits) return 2;
    const size_t degree = (size_t)1 << degree_bits;
    const size_t step = (size_t)1 << (rate_bits - quotient_degree_bits);
    const size_t next_step = (size_t)1 << quotient_degree_bits;
    const size_t lde_size = degree << quotient_degree_bits;
    // ZeroPolyOnCoset::new(degree_bits, quotient_degree_bits)
    u64 g_pow_n = MULTIPLICATIVE_GROUP_GENERATOR;
    for (uint32_t k = 0; k < degree_bits; k++) g_pow_n = fsqr(g_pow_n);
    const size_t rate = (size_t)1 << quotient_degree_bits;
    std::vector<u64> zh_evals(rate), zh_inverses(rate);
    {
        u64 w = primitive_root_of_unity(quotient_degree_bits), x = 1;
        for (size_t j = 0; j < rate; j++) {
            zh_evals[j] = fsub(fmul(g_pow_n, x), 1);
            zh_inverses[j] = finv(zh_evals[j]);
            x = fmul(x, w);
        }
    }
    const u64 n_field = canon((u64)degree);
    const u64 w_lde = primitive_root_of_unity(degree_bits + quotient_degree_bits);
    std::vector<u64> points(lde_size);  // two_adic_subgroup
    {
        u64 x = 1;
        for (size_t i = 0; i < lde_size; i++) {
            points[i] = x;
            x = fmul(x, w_lde);
        }
    }
    std::vector<u64> quotient_values(lde_size * num_challenges);
    std::vector<u64> local_constants_sigmas(constants_sigmas->B), local_wires(wires->B), local_zs(zs_partial_products->B),
        next_zs(zs_partial_products->B), gate_res, constraint_terms(cd->num_gate_constraints), vanishing_terms;
    for (size_t i = 0; i < lde_size; i++) {
        const u64 shifted_x = fmul(MULTIPLICATIVE_GROUP_GENERATOR, points[i]);
        const size_t i_next = (i + next_step) % lde_size;
        glo_commit_get_lde_values(constants_sigmas, i, step, local_constants_sigmas.data());
        glo_commit_get_lde_values(wires, i, step, local_wires.data());
        glo_commit_get_lde_values(zs_partial_products, i, step, local_zs.data());
        glo_commit_get_lde_values(zs_partial_products, i_next, step, next_zs.data());
        const u64* local_constants = local_constants_sigmas.data();              // constants_range
        const u64* s_sigmas = local_constants_sigmas.data() + cd->num_constants;  // sigmas_range
        const u64* partial_products = local_zs.data() + num_challenges;           // partial_products_range
        // evaluate_gate_constraints_base_batch
        std::fill(constraint_terms.begin(), constraint_terms.end(), 0);
        for (size_t gi = 0; gi < cd->n_gates; gi++) {
            const glo_gate& g = cd->gates[gi];
            const u64 s = local_constants[g.selector_index];
            u64 filter = 1;  // compute_filter
            for (size_t j = g.group_start; j < g.group_end; j++)
                if (j != gi) filter = fmul(filter, fsub(canon((u64)j), s));
            if (cd->num_selectors > 1) filter = fmul(filter, fsub(UNUSED_SELECTOR, s));
            gate_eval_unfiltered(g, local_constants + cd->num_selectors + cd->num_lookup_selectors, local_wires.data(),
                                 public_inputs_hash, gate_res);
            if (gate_res.size() > constraint_terms.size()) return 5;  // "num_constraints() gave too low of a number"
            for (size_t j = 0; j < gate_res.size(); j++) constraint_terms[j] = fadd(constraint_terms[j], fmul(gate_res[j], filter));
        }
        vanishing_terms.clear();
        const u64 l_0_x = fmul(zh_evals[i % rate], finv(fmul(n_field, fsub(shifted_x, 1))));  // eval_l_0
        std::vector<u64> vanishing_partial_products_terms, vanishing_all_lookup_terms;
        for (size_t c = 0; c < num_challenges; c++) {
            const u64 z_x = local_zs[c], z_gx = next_zs[c];
            vanishing_terms.push_back(fmul(l_0_x, fsub(z_x, 1)));  // vanishing_z_1_terms
            if (has_lookup) {
                const size_t at = num_challenges * (1 + num_prods) + cd->num_lookup_polys * c;  // lookup_range
                check_lookup_constraints_batch(cd, local_wires.data(), local_zs.data() + at, next_zs.data() + at,
                                               local_constants + cd->num_selectors, deltas + 4 * c, lut_re_poly_evals[c],
                                               vanishing_all_lookup_terms);
            }
            std::vector<u64> numerator_values(num_routed_wires), denominator_values(num_routed_wires);
            for (size_t j = 0; j < num_routed_wires; j++) {
                const u64 wire_value = local_wires[j];
                const u64 s_id = fmul(cd->k_is[j], shifted_x);
                numerator_values[j] = fadd(fadd(wire_value, fmul(betas[c], s_id)), gammas[c]);
                denominator_values[j] = fadd(fadd(wire_value, fmul(betas[c], s_sigmas[j])), gammas[c]);
            }
            // check_partial_products
            const u64* current_partial_products = partial_products + c * num_prods;
            for (size_t k = 0; k * max_degree < num_routed_wires; k++) {
                const size_t lo = k * max_degree, hi = std::min(lo + max_degree, num_routed_wires);
                u64 num_chunk_product = 1, den_chunk_product = 1;
                for (size_t j = lo; j < hi; j++) {
                    num_chunk_product = fmul(num_chunk_product, numerator_values[j]);
                    den_chunk_product = fmul(den_chunk_product, denominator_values[j]);
                }
                const u64 prev_acc = k == 0 ? z_x : current_partial_products[k - 1];
                const u64 next_acc = k == num_prods ? z_gx : current_partial_products[k];
                vanishing_partial_products_terms.push_back(fsub(fmul(prev_acc, num_chunk_product), fmul(next_acc, den_chunk_product)));
            }
        }
        vanishing_terms.insert(vanishing_terms.end(), vanishing_partial_products_terms.begin(), vanishing_partial_products_terms.end());
        vanishing_terms.insert(vanishing_terms.end(), vanishing_all_lookup_terms.begin(), vanishing_all_lookup_terms.end());
        vanishing_terms.insert(vanishing_terms.end(), constraint_terms.begin(), constraint_terms.end());
        const u64 denominator_inv = zh_inverses[i % rate];
        for (size_t c = 0; c < num_challenges; c++) {  // reduce_with_powers_multi
            u64 cumul = 0;
            for (size_t t = vanishing_terms.size(); t-- > 0;) cumul = fadd(fmul(cumul, alphas[c]), vanishing_terms[t]);
            quotient_values[i * num_challenges + c] = fmul(cumul, denominator_inv);
        }
    }
    for (size_t c = 0; c < num_challenges; c++) {  // transpose + coset_ifft
        u64* col = out + c * lde_size;
        for (size_t i = 0; i < lde_size; i++) col[i] = quotient_values[i * num_challenges + c];
        coset_ifft(col, lde_size, MULTIPLICATIVE_GROUP_GENERATOR);
        for (size_t i = 0; i < lde_size; i++) col[i] = canon(col[i]);
    }
    return 0;
}

void glo_eval_poly_base_at_ext(const uint64_t* coeffs, size_t n, const uint64_t z[2], uint64_t out[2]) {
    E2 zz{z[0], z[1]}, acc = e2(0);
    for (size_t k = n; k-- > 0;) acc = eadd(emul(acc, zz), e2(coeffs[k]));
    out[0] = canon(acc.a);
    out[1] = canon(acc.b);
}

// prove_openings (oracle.rs:176-237) -> fri_proof (prover.rs:24-70)
int glo_prove_openings(const glo_commit* const* oracles, size_t n_oracles, const glo_fri_batch* batches,
                       size_t n_batches, glo_challenger* ch, const glo_fri_params* params, uint8_t** out,
                       size_t* out_len, uint64_t* tap_final_poly, uint64_t* tap_betas,
                       uint64_t* tap_pow_witness, uint64_t* tap_query_indices) {
    if (n_oracles == 0) return 1;
    size_t n = oracles[0]->n;
    uint32_t rate_bits = params->rate_bits;
    // alpha = challenger.get_extension_challenge()                     oracle.rs:186
    E2 alpha = get_extension_challenge(ch);
    u64 alpha_count = 0;  // ReducingFactor.count
    std::vector<E2> final_poly;  // PolynomialCoeffs::empty()
    for (size_t bi = 0; bi < n_batches; bi++) {
        const glo_fri_batch& batch = batches[bi];
        E2 point{batch.point[0], batch.point[1]};
        // composition_poly = alpha.reduce_polys_base(polys_coeff)     reducing.rs:83-95
        std::vector<E2> comp(n, e2(0));
        E2 base_power = e2(1);
        for (size_t j = 0; j < batch.num_polys; j++) {
            const glo_commit* oc = oracles[batch.oracle_index[j]];
            if (oc->n != n) return 2;
            const u64* poly = oc->coeffs.data() + (size_t)batch.poly_index[j] * n;
            alpha_count++;
            for (size_t k = 0; k < n; k++) comp[k] = eadd(comp[k], escale(base_power, poly[k]));
            base_power = emul(base_power, alpha);
        }
        // quotient = composition_poly.divide_by_linear(point)         division.rs:75-88
        std::vector<E2> bs(n);
        E2 acc = e2(0);
        for (size_t k = n; k-- > 0;) {
            acc = eadd(emul(acc, point), comp[k]);
            bs[n - 1 - k] = acc;  // scan over reversed coefficients
        }
        bs.pop_back();
        std::reverse(bs.begin(), bs.end());
        bs.push_back(e2(0));  // pad back to power of two             oracle.rs:210
        // alpha.shift_poly(&mut final_poly); final_poly += quotient   reducing.rs:102-106
        E2 sh = eexp(alpha, alpha_count);
        alpha_count = 0;
        if (final_poly.empty()) {
            final_poly = bs;
        } else {
            for (size_t k = 0; k < n; k++) final_poly[k] = eadd(emul(final_poly[k], sh), bs[k]);
        }
    }
    if (tap_final_poly)
        for (size_t k = 0; k < n; k++) {
            tap_final_poly[2 * k] = canon(final_poly[k].a);
            tap_final_poly[2 * k + 1] = canon(final_poly[k].b);
        }
    // lde_final_poly = final_poly.lde(rate_bits); values = coset_fft(coset_shift)   oracle.rs:215-220
    size_t N = n << rate_bits;
    std::vector<E2> coeffs(N, e2(0));
    for (size_t k = 0; k < n; k++) coeffs[k] = final_poly[k];
    std::vector<E2> values = coeffs;
    ext_coset_fft(values, MULTIPLICATIVE_GROUP_GENERATOR);

    // ---- fri_committed_trees, prover.rs:84-150
    std::vector<Tree> trees;
    u64 shift = MULTIPLICATIVE_GROUP_GENERATOR;
    for (uint32_t round = 0; round < params->num_reductions; round++) {
        uint32_t arity_bits = params->reduction_arity_bits[round];
        size_t arity = (size_t)1 << arity_bits;
        // reverse_index_bits_in_place(&mut values.values); chunks(arity).map(flatten)
        std::vector<u64> flat(values.size() * 2);
        for (size_t i = 0; i < values.size(); i++) {
            flat[2 * i] = canon(values[i].a);
            flat[2 * i + 1] = canon(values[i].b);
        }
        reverse_index_bits_in_place(flat.data(), values.size(), 2);
        Tree t;
        t.N = values.size() / arity;
        t.W = 2 * arity;
        t.cap_height = params->cap_height;
        if (t.cap_height > log2_strict(t.N)) return 3;
        size_t C = (size_t)1 << t.cap_height;
        t.leaves = std::move(flat);
        t.digests.resize(2 * (t.N - C));
        t.cap.resize(C);
        merkle_build(t.leaves.data(), t.N, t.W, t.cap_height, t.digests.data(), t.cap.data(), 8);
        observe_cap(ch, t.cap);
        trees.push_back(std::move(t));
        E2 beta = get_extension_challenge(ch);
        if (tap_betas) {
            tap_betas[2 * round] = beta.a;
            tap_betas[2 * round + 1] = beta.b;
        }
        // coeffs = chunks_exact(arity).map(|chunk| reduce_with_powers(chunk, beta))   plonk_common.rs:118-130
        std::vector<E2> folded(coeffs.size() / arity);
        for (size_t j = 0; j < folded.size(); j++) {
            E2 sum = e2(0);
            for (size_t i = arity; i-- > 0;) sum = eadd(emul(sum, beta), coeffs[arity * j + i]);
            folded[j] = sum;
        }
        coeffs = std::move(folded);
        shift = fexp(shift, arity);
        values = coeffs;
        ext_coset_fft(values, shift);
    }
    // truncate; observe final coefficients                             prover.rs:134-147
    coeffs.resize(coeffs.size() >> rate_bits);
    for (auto& c : coeffs) observe_ext(ch, c);

    // ---- fri_proof_of_work, prover.rs:153-202 (smallest qualifying nonce)
    uint32_t min_leading_zeros = params->proof_of_work_bits + (64 - 64);
    u64 inter[12];
    memcpy(inter, ch->sponge_state, sizeof(inter));
    size_t witness_input_pos = ch->input_buffer.size();
    for (size_t i = 0; i < witness_input_pos; i++) inter[i] = ch->input_buffer[i];
    u64 pow_witness = 0;
    for (u64 cand = 0;; cand++) {
        u64 st[12];
        memcpy(st, inter, sizeof(st));
        st[witness_input_pos] = cand;
        poseidon(st);
        u64 resp = canon(st[7]);  // squeeze().last()
        uint32_t lz = resp == 0 ? 64 : (uint32_t)__builtin_clzll(resp);
        if (lz >= min_leading_zeros) {
            pow_witness = cand;
            break;
        }
        if (cand == P - 1) return 4;
    }
    observe_element(ch, pow_witness);
    u64 pow_response = get_challenge(ch);
    {
        uint32_t lz = pow_response == 0 ? 64 : (uint32_t)__builtin_clzll(pow_response);
        if (lz < min_leading_zeros) return 5;
    }
    if (tap_pow_witness) *tap_pow_witness = pow_witness;

    // ---- serialise: write_fri_proof, serialization/mod.rs:1595-1609
    std::vector<uint8_t> buf;
    for (auto& t : trees)
        for (auto& h : t.cap) put_hash(buf, h);
    // fri_prover_query_rounds, prover.rs:204-258
    for (uint32_t q = 0; q < params->num_query_rounds; q++) {
        u64 rand = get_challenge(ch);
        size_t x_index = (size_t)(rand % N);
        if (tap_query_indices) tap_query_indices[q] = x_index;
        for (size_t o = 0; o < n_oracles; o++) {
            const glo_commit* oc = oracles[o];
            const u64* leaf = oc->leaves.data() + x_index * oc->W;
            for (size_t i = 0; i < oc->W; i++) put_u64(buf, leaf[i]);
            size_t len = log2_strict(oc->N) - oc->cap_height;
            std::vector<Hash> sib(len);
            merkle_prove(x_index, oc->N, oc->cap_height, oc->digests.data(), sib.data());
            buf.push_back((uint8_t)len);
            for (auto& h : sib) put_hash(buf, h);
        }
        for (size_t i = 0; i < trees.size(); i++) {
            uint32_t arity_bits = params->reduction_arity_bits[i];
            const Tree& t = trees[i];
            size_t idx = x_index >> arity_bits;
            const u64* leaf = t.leaves.data() + idx * t.W;
            for (size_t k = 0; k < t.W; k++) put_u64(buf, leaf[k]);
            size_t len = log2_strict(t.N) - t.cap_height;
            std::vector<Hash> sib(len);
            merkle_prove(idx, t.N, t.cap_height, t.digests.data(), sib.data());
            buf.push_back((uint8_t)len);
            for (auto& h : sib) put_hash(buf, h);
            x_index >>= arity_bits;
        }
    }
    for (auto& c : coeffs) {
        put_u64(buf, c.a);
        put_u64(buf, c.b);
    }
    put_u64(buf, pow_witness);
    *out = (uint8_t*)malloc(buf.size());
    memcpy(*out, buf.data(), buf.size());
    *out_len = buf.size();
    return 0;
}

glo_batch_commit* glo_batch_commit_new(const uint64_t* const* polys, const uint32_t* log_lens, size_t num_polys,
                                       uint32_t rate_bits, uint32_t cap_height, int is_coeffs) {
    for (size_t i = 0; i + 1 < num_polys; i++)
        if (log_lens[i] < log_lens[i + 1]) return nullptr;  // assert!(degree_bits.windows(2).all(|p| p[0] >= p[1]))
    glo_batch_commit* c = new glo_batch_commit();
    c->rate_bits = rate_bits;
    c->cap_height = cap_height;
    size_t group_start = 0;
    for (size_t i = 0; i < num_polys; i++) {
        if (i == num_polys - 1 || log_lens[i] > log_lens[i + 1]) {
            glo_batch_commit::Group g;
            g.degree_bits = log_lens[i];
            g.B = i + 1 - group_start;
            g.n = (size_t)1 << g.degree_bits;
            g.N = g.n << rate_bits;
            g.coeffs.resize(g.B * g.n);
            std::vector<u64> lde(g.N);
            g.leaves.resize(g.N * g.B);
            const uint32_t lgN = g.degree_bits + rate_bits;
            for (size_t b = 0; b < g.B; b++) {
                u64* co = g.coeffs.data() + b * g.n;
                memcpy(co, polys[group_start + b], g.n * 8);
                if (!is_coeffs) ifft_with_options(co, g.n, nullptr);  // values.map(|v| v.ifft())
                for (size_t k = 0; k < g.n; k++) co[k] = canon(co[k]);
                // PolynomialBatch::lde_values (oracle.rs:114-139): lde + coset_fft
                memcpy(lde.data(), co, g.n * 8);
                memset(lde.data() + g.n, 0, (g.N - g.n) * 8);
                coset_fft_with_options(lde.data(), g.N, MULTIPLICATIVE_GROUP_GENERATOR, rate_bits, nullptr);
                // transpose + reverse_index_bits_in_place (oracle.rs:104-106)
                for (size_t j = 0; j < g.N; j++) g.leaves[(size_t)reverse_bits(j, lgN) * g.B + b] = canon(lde[j]);
                c->where.emplace_back(c->groups.size(), b);
            }
            c->groups.push_back(std::move(g));
            group_start = i + 1;
        }
    }
    // BatchMerkleTree::new: a chain of fill_digests_buf calls, cap of stage k = number of leaves of stage k+1
    std::vector<Hash> cap;
    for (size_t k = 0; k < c->groups.size(); k++) {
        const glo_batch_commit::Group& g = c->groups[k];
        glo_batch_commit::Stage st;
        st.N = g.N;
        st.cap_height = k + 1 < c->groups.size() ? c->groups[k + 1].degree_bits + rate_bits : cap_height;
        if (st.cap_height > log2_strict(st.N) || (k + 1 < c->groups.size() && st.cap_height >= log2_strict(st.N))) {
            delete c;
            return nullptr;
        }
        if (k == 0) {
            st.W = g.B;
            st.rows = g.leaves;
        } else {  // new_leaves = cap_hash.to_vec() ++ cur[i]   (batch_merkle_tree.rs:85-96)
            st.W = 4 + g.B;
            st.rows.resize(st.N * st.W);
            for (size_t i = 0; i < st.N; i++) {
                memcpy(st.rows.data() + i * st.W, cap[i].e, 32);
                memcpy(st.rows.data() + i * st.W + 4, g.leaves.data() + i * g.B, g.B * 8);
            }
        }
        const size_t C = (size_t)1 << st.cap_height;
        st.digests.resize(2 * (st.N - C));
        st.cap.resize(C);
        merkle_build(st.rows.data(), st.N, st.W, st.cap_height, st.digests.data(), st.cap.data(), 8);
        cap = st.cap;
        c->stages.push_back(std::move(st));
    }
    return c;
}
void glo_batch_commit_free(glo_batch_commit* c) { delete c; }
size_t glo_batch_commit_cap(const glo_batch_commit* c, uint64_t* out) {
    const std::vector<Hash>& cap = c->stages.back().cap;
    if (out) memcpy(out, cap.data(), cap.size() * 32);
    return cap.size();
}

// BatchFriOracle::prove_openings + batch_fri_proof (batch_fri/oracle.rs:124-183, batch_fri/prover.rs:30-215), serialised
// like write_fri_proof. instances[i] = the opening batches of the polynomials of degree 2^degree_bits[i].
int glo_batch_prove_openings(const glo_batch_commit* const* oracles, size_t n_oracles, const uint32_t* degree_bits,
                             const glo_fri_instance* instances, size_t n_instances, glo_challenger* ch,
                             const glo_fri_params* params, uint8_t** out, size_t* out_len) {
    if (n_oracles == 0 || n_instances == 0) return 1;
    const uint32_t rate_bits = params->rate_bits;
    E2 alpha = get_extension_challenge(ch);
    std::vector<std::vector<E2>> lde_coeffs, lde_values;
    for (size_t ii = 0; ii < n_instances; ii++) {
        const size_t n = (size_t)1 << degree_bits[ii];
        u64 alpha_count = 0;
        std::vector<E2> final_poly;
        for (size_t bi = 0; bi < instances[ii].n_batches; bi++) {
            const glo_fri_batch& batch = instances[ii].batches[bi];
            E2 point{batch.point[0], batch.point[1]};
            std::vector<E2> comp(n, e2(0));
            E2 base_power = e2(1);
            for (size_t j = 0; j < batch.num_polys; j++) {
                const glo_batch_commit* oc = oracles[batch.oracle_index[j]];
                const auto wh = oc->where[batch.poly_index[j]];
                const glo_batch_commit::Group& g = oc->groups[wh.first];
                if (g.n != n) return 2;
                const u64* poly = g.coeffs.data() + wh.second * n;
                alpha_count++;
                for (size_t k = 0; k < n; k++) comp[k] = eadd(comp[k], escale(base_power, poly[k]));
                base_power = emul(base_power, alpha);
            }
            std::vector<E2> bs(n);
            E2 acc = e2(0);
            for (size_t k = n; k-- > 0;) {
                acc = eadd(emul(acc, point), comp[k]);
                bs[n - 1 - k] = acc;
            }
            bs.pop_back();
            std::reverse(bs.begin(), bs.end());
            bs.push_back(e2(0));
            E2 sh = eexp(alpha, alpha_count);
            alpha_count = 0;
            if (final_poly.empty()) final_poly = bs;
            else
                for (size_t k = 0; k < n; k++) final_poly[k] = eadd(emul(final_poly[k], sh), bs[k]);
        }
        if (final_poly.size() != n) return 3;  // assert_eq!(final_poly.len(), 1 << degree_bits[i])
        std::vector<E2> co(n << rate_bits, e2(0));
        for (size_t k = 0; k < n; k++) co[k] = final_poly[k];
        std::vector<E2> va = co;
        ext_coset_fft(va, MULTIPLICATIVE_GROUP_GENERATOR);
        lde_coeffs.push_back(std::move(co));
        lde_values.push_back(std::move(va));
    }
    // batch_fri_proof's shape checks (prover.rs:38-57)
    const size_t N = lde_coeffs[0].size();
    for (size_t i = 0; i + 1 < lde_values.size(); i++)
        if (lde_values[i].size() <= lde_values[i + 1].size()) return 4;
    // batch_fri_committed_trees (prover.rs:88-147)
    std::vector<Tree> trees;
    std::vector<E2> final_coeffs = lde_coeffs[0], final_values = lde_values[0];
    u64 shift = MULTIPLICATIVE_GROUP_GENERATOR;
    size_t polynomial_index = 1;
    for (uint32_t round = 0; round < params->num_reductions; round++) {
        const uint32_t arity_bits = params->reduction_arity_bits[round];
        const size_t arity = (size_t)1 << arity_bits;
        std::vector<u64> flat(final_values.size() * 2);
        for (size_t i = 0; i < final_values.size(); i++) {
            flat[2 * i] = canon(final_values[i].a);
            flat[2 * i + 1] = canon(final_values[i].b);
        }
        reverse_index_bits_in_place(flat.data(), final_values.size(), 2);
        Tree t;
        t.N = final_values.size() / arity;
        t.W = 2 * arity;
        t.cap_height = params->cap_height;
        if (t.cap_height > log2_strict(t.N)) return 5;
        const size_t C = (size_t)1 << t.cap_height;
        t.leaves = std::move(flat);
        t.digests.resize(2 * (t.N - C));
        t.cap.resize(C);
        merkle_build(t.leaves.data(), t.N, t.W, t.cap_height, t.digests.data(), t.cap.data(), 8);
        observe_cap(ch, t.cap);
        trees.push_back(std::move(t));
        const E2 beta = get_extension_challenge(ch);
        std::vector<E2> folded(final_coeffs.size() / arity);
        for (size_t j = 0; j < folded.size(); j++) {
            E2 sum = e2(0);
            for (size_t i = arity; i-- > 0;) sum = eadd(emul(sum, beta), final_coeffs[arity * j + i]);
            folded[j] = sum;
        }
        final_coeffs = std::move(folded);
        shift = fexp(shift, arity);
        final_values = final_coeffs;
        ext_coset_fft(final_values, shift);
        if (polynomial_index != lde_values.size() && final_values.size() == lde_values[polynomial_index].size()) {
            for (size_t i = 0; i < final_values.size(); i++)
                final_values[i] = eadd(emul(final_values[i], beta), lde_values[polynomial_index][i]);
            polynomial_index++;
        }
        final_coeffs = final_values;
        ext_coset_ifft(final_coeffs, shift);
    }
    if (polynomial_index != lde_values.size()) return 6;
    final_coeffs.resize(final_coeffs.size() >> rate_bits);
    for (auto& cf : final_coeffs) observe_ext(ch, cf);
    // fri_proof_of_work (smallest qualifying nonce)
    const uint32_t min_leading_zeros = params->proof_of_work_bits;
    u64 inter[12];
    memcpy(inter, ch->sponge_state, sizeof(inter));
    const size_t witness_input_pos = ch->input_buffer.size();
    for (size_t i = 0; i < witness_input_pos; i++) inter[i] = ch->input_buffer[i];
    u64 pow_witness = 0;
    for (u64 cand = 0;; cand++) {
        u64 st[12];
        memcpy(st, inter, sizeof(st));
        st[witness_input_pos] = cand;
        poseidon(st);
        const u64 resp = canon(st[7]);
        const uint32_t lz = resp == 0 ? 64 : (uint32_t)__builtin_clzll(resp);
        if (lz >= min_leading_zeros) {
            pow_witness = cand;
            break;
        }
    }
    observe_element(ch, pow_witness);
    (void)get_challenge(ch);
    // serialise (write_fri_proof); batch_fri_prover_query_round (prover.rs:171-215)
    std::vector<uint8_t> buf;
    for (auto& t : trees)
        for (auto& h : t.cap) put_hash(buf, h);
    for (uint32_t q = 0; q < params->num_query_rounds; q++) {
        size_t x_index = (size_t)(get_challenge(ch) % N);
        for (size_t o = 0; o < n_oracles; o++) {
            const glo_batch_commit* oc = oracles[o];
            const uint32_t h0 = oc->groups[0].degree_bits + rate_bits;
            // t.values(x_index).flatten()
            for (const auto& g : oc->groups) {
                const size_t idx = x_index >> (h0 - (g.degree_bits + rate_bits));
                for (size_t i = 0; i < g.B; i++) put_u64(buf, g.leaves[idx * g.B + i]);
            }
            // t.open_batch(x_index): the stages' sibling paths back to back
            std::vector<Hash> sib;
            for (const auto& st : oc->stages) {
                const uint32_t hk = log2_strict(st.N);
                const size_t len = hk - st.cap_height;
                std::vector<Hash> part(len);
                merkle_prove(x_index >> (h0 - hk), st.N, st.cap_height, st.digests.data(), part.data());
                sib.insert(sib.end(), part.begin(), part.end());
            }
            buf.push_back((uint8_t)sib.size());
            for (auto& h : sib) put_hash(buf, h);
        }
        for (size_t i = 0; i < trees.size(); i++) {
            const uint32_t arity_bits = params->reduction_arity_bits[i];
            const Tree& t = trees[i];
            const size_t idx = x_index >> arity_bits;
            const u64* leaf = t.leaves.data() + idx * t.W;
            for (size_t k = 0; k < t.W; k++) put_u64(buf, leaf[k]);
            const size_t len = log2_strict(t.N) - t.cap_height;
            std::vector<Hash> sib(len);
            merkle_prove(idx, t.N, t.cap_height, t.digests.data(), sib.data());
            buf.push_back((uint8_t)len);
            for (auto& h : sib) put_hash(buf, h);
            x_index >>= arity_bits;
        }
    }
    for (auto& cf : final_coeffs) {
        put_u64(buf, cf.a);
        put_u64(buf, cf.b);
    }
    put_u64(buf, pow_witness);
    *out = (uint8_t*)malloc(buf.size());
    memcpy(*out, buf.data(), buf.size());
    *out_len = buf.size();
    return 0;
}

// verify_batch_fri_proof, batch_fri/verifier.rs:22-251 (+ verify_batch_merkle_proof_to_cap, hash/merkle_proofs.rs:72-107;
// challenges as in fri_challenges, fri/challenges.rs:28-75). group_num_polys[o * n_instances + i] = polynomials of oracle o
// in degree group i (FriInstanceInfo.oracles[o].num_polys of instance i). opened_values: per instance, per batch, per
// polynomial (2 words). Returns 0 if the proof verifies.
int glo_verify_batch_fri_proof(const uint64_t* const* initial_caps, const size_t* group_num_polys, size_t n_oracles,
                               const uint32_t* degree_bits, const glo_fri_instance* instances, size_t n_instances,
                               const uint64_t* opened_values, glo_challenger* ch, const glo_fri_params* params,
                               const uint8_t* proof, size_t proof_len) {
    size_t pos = 0;
    bool overrun = false;
    auto get_u64 = [&]() -> u64 {
        if (pos + 8 > proof_len) {
            overrun = true;
            return 0;
        }
        u64 v = 0;
        for (int i = 0; i < 8; i++) v |= (u64)proof[pos + i] << (8 * i);
        pos += 8;
        return v;
    };
    auto get_hash = [&]() {
        Hash h;
        for (int i = 0; i < 4; i++) h.e[i] = get_u64();
        return h;
    };
    const uint32_t rate_bits = params->rate_bits;
    std::vector<uint32_t> heights(n_instances);  // degree_bits + rate_bits
    for (size_t i = 0; i < n_instances; i++) heights[i] = degree_bits[i] + rate_bits;
    const uint32_t log_N = heights[0];
    const size_t N = (size_t)1 << log_N;
    const size_t C = (size_t)1 << params->cap_height;
    const uint32_t R = params->num_reductions;
    std::vector<std::vector<Hash>> caps(R, std::vector<Hash>(C));
    for (uint32_t r = 0; r < R; r++)
        for (size_t c = 0; c < C; c++) caps[r][c] = get_hash();
    struct Query {
        std::vector<std::vector<u64>> init_leaf;
        std::vector<std::vector<Hash>> init_sib;
        std::vector<std::vector<E2>> evals;
        std::vector<std::vector<Hash>> step_sib;
    };
    std::vector<Query> queries(params->num_query_rounds);
    for (auto& q : queries) {
        for (size_t o = 0; o < n_oracles; o++) {
            size_t width = 0;
            for (size_t i = 0; i < n_instances; i++) width += group_num_polys[o * n_instances + i];
            std::vector<u64> leaf(width);
            for (auto& x : leaf) x = get_u64();
            if (pos >= proof_len) return 10;
            size_t len = proof[pos++];
            std::vector<Hash> sib(len);
            for (auto& h : sib) h = get_hash();
            q.init_leaf.push_back(leaf);
            q.init_sib.push_back(sib);
        }
        for (uint32_t r = 0; r < R; r++) {
            size_t arity = (size_t)1 << params->reduction_arity_bits[r];
            std::vector<E2> ev(arity);
            for (auto& e : ev) {
                e.a = get_u64();
                e.b = get_u64();
            }
            if (pos >= proof_len) return 10;
            size_t len = proof[pos++];
            std::vector<Hash> sib(len);
            for (auto& h : sib) h = get_hash();
            q.evals.push_back(ev);
            q.step_sib.push_back(sib);
        }
    }
    uint32_t final_bits = degree_bits[0];
    for (uint32_t r = 0; r < R; r++) final_bits -= params->reduction_arity_bits[r];
    std::vector<E2> final_poly((size_t)1 << final_bits);
    for (auto& c : final_poly) {
        c.a = get_u64();
        c.b = get_u64();
    }
    const u64 pow_witness = get_u64();
    if (overrun || pos != proof_len) return 10;
    // fri_challenges
    const E2 fri_alpha = get_extension_challenge(ch);
    std::vector<E2> betas;
    for (uint32_t r = 0; r < R; r++) {
        observe_cap(ch, caps[r]);
        betas.push_back(get_extension_challenge(ch));
    }
    for (auto& c : final_poly) observe_ext(ch, c);
    observe_element(ch, pow_witness);
    const u64 pow_response = get_challenge(ch);
    std::vector<size_t> indices;
    for (uint32_t q = 0; q < params->num_query_rounds; q++) indices.push_back((size_t)(get_challenge(ch) % N));
    {
        const uint32_t lz = pow_response == 0 ? 64 : (uint32_t)__builtin_clzll(pow_response);
        if (lz < params->proof_of_work_bits) return 11;
    }
    // PrecomputedReducedOpenings per instance
    std::vector<std::vector<E2>> reduced(n_instances);
    {
        size_t off = 0;
        for (size_t i = 0; i < n_instances; i++)
            for (size_t b = 0; b < instances[i].n_batches; b++) {
                const glo_fri_batch& batch = instances[i].batches[b];
                E2 acc = e2(0);
                for (size_t j = batch.num_polys; j-- > 0;)
                    acc = eadd(emul(acc, fri_alpha), E2{opened_values[2 * (off + j)], opened_values[2 * (off + j) + 1]});
                off += batch.num_polys;
                reduced[i].push_back(acc);
            }
    }
    // batch_fri_combine_initial (verifier.rs:105-144)
    auto combine_initial = [&](const Query& q, size_t inst, u64 subgroup_x) {
        E2 sum = e2(0);
        u64 count = 0;
        for (size_t b = 0; b < instances[inst].n_batches; b++) {
            const glo_fri_batch& batch = instances[inst].batches[b];
            const E2 point{batch.point[0], batch.point[1]};
            E2 red = e2(0);
            for (size_t j = batch.num_polys; j-- > 0;) {
                const u64 ev = q.init_leaf[batch.oracle_index[j]][batch.poly_index[j]];  // unsalted_eval
                red = eadd(emul(red, fri_alpha), e2(ev));
                count++;
            }
            const E2 numerator = esub(red, reduced[inst][b]);
            const E2 denominator = esub(e2(subgroup_x), point);
            sum = emul(eexp(fri_alpha, count), sum);
            count = 0;
            sum = eadd(sum, emul(numerator, einv(denominator)));
        }
        return sum;
    };
    for (size_t qi = 0; qi < queries.size(); qi++) {
        const Query& q = queries[qi];
        size_t x_index = indices[qi];
        // batch_fri_verify_initial_proof (verifier.rs:75-103) + verify_batch_merkle_proof_to_cap
        for (size_t o = 0; o < n_oracles; o++) {
            size_t leaf_off = 0, leaf_index = x_index;
            Hash cur = hash_or_noop(q.init_leaf[o].data(), group_num_polys[o * n_instances + 0]);
            leaf_off += group_num_polys[o * n_instances + 0];
            uint32_t current_height = heights[0];
            size_t leaf_data_index = 1;
            for (const Hash& sib : q.init_sib[o]) {
                const size_t bit = leaf_index & 1;
                leaf_index >>= 1;
                cur = bit ? two_to_one(sib, cur) : two_to_one(cur, sib);
                current_height -= 1;
                if (leaf_data_index < n_instances && current_height == heights[leaf_data_index]) {
                    const size_t w = group_num_polys[o * n_instances + leaf_data_index];
                    std::vector<u64> nl(cur.e, cur.e + 4);
                    nl.insert(nl.end(), q.init_leaf[o].begin() + leaf_off, q.init_leaf[o].begin() + leaf_off + w);
                    cur = hash_or_noop(nl.data(), nl.size());
                    leaf_off += w;
                    leaf_data_index++;
                }
            }
            if (leaf_data_index != n_instances) return 12;
            if (!heq(cur, ((const Hash*)initial_caps[o])[leaf_index])) return 13;
        }
        uint32_t n = heights[0];
        u64 subgroup_x = fmul(MULTIPLICATIVE_GROUP_GENERATOR, fexp(primitive_root_of_unity(n), reverse_bits(x_index, n)));
        size_t batch_index = 0;
        E2 old_eval = combine_initial(q, batch_index, subgroup_x);
        batch_index++;
        for (uint32_t r = 0; r < R; r++) {
            const uint32_t arity_bits = params->reduction_arity_bits[r];
            const size_t arity = (size_t)1 << arity_bits;
            const std::vector<E2>& evals = q.evals[r];
            const size_t coset_index = x_index >> arity_bits, within = x_index & (arity - 1);
            if (!eeq(evals[within], old_eval)) return 14;
            {  // compute_evaluation, fri/verifier.rs:22-47
                const u64 g = primitive_root_of_unity(arity_bits);
                std::vector<E2> ev = evals;
                std::vector<u64> flat(2 * arity);
                for (size_t i = 0; i < arity; i++) {
                    flat[2 * i] = ev[i].a;
                    flat[2 * i + 1] = ev[i].b;
                }
                reverse_index_bits_in_place(flat.data(), arity, 2);
                for (size_t i = 0; i < arity; i++) ev[i] = E2{flat[2 * i], flat[2 * i + 1]};
                const size_t rev_within = reverse_bits(within, arity_bits);
                const u64 coset_start = fmul(subgroup_x, fexp(g, arity - rev_within));
                std::vector<E2> xs(arity);
                u64 y = 1;
                for (size_t i = 0; i < arity; i++) {
                    xs[i] = e2(fmul(coset_start, y));
                    y = fmul(y, g);
                }
                const E2 beta = betas[r];
                E2 result = e2(0);
                bool hit = false;
                for (size_t i = 0; i < arity; i++)
                    if (eeq(xs[i], beta)) {
                        result = ev[i];
                        hit = true;
                    }
                if (!hit) {
                    E2 l_x = e2(1);
                    for (size_t i = 0; i < arity; i++) l_x = emul(l_x, esub(beta, xs[i]));
                    E2 sacc = e2(0);
                    for (size_t i = 0; i < arity; i++) {
                        E2 w = e2(1);
                        for (size_t j = 0; j < arity; j++)
                            if (j != i) w = emul(w, esub(xs[i], xs[j]));
                        sacc = eadd(sacc, emul(emul(einv(w), einv(esub(beta, xs[i]))), ev[i]));
                    }
                    result = emul(l_x, sacc);
                }
                old_eval = result;
            }
            std::vector<u64> flat(2 * arity);
            for (size_t i = 0; i < arity; i++) {
                flat[2 * i] = evals[i].a;
                flat[2 * i + 1] = evals[i].b;
            }
            if (!merkle_verify(flat.data(), flat.size(), coset_index, q.step_sib[r].data(), q.step_sib[r].size(), caps[r].data()))
                return 15;
            for (uint32_t k = 0; k < arity_bits; k++) subgroup_x = fsqr(subgroup_x);
            x_index = coset_index;
            n -= arity_bits;
            if (batch_index < n_instances && n == heights[batch_index]) {
                const u64 subgroup_x_init =
                    fmul(MULTIPLICATIVE_GROUP_GENERATOR, fexp(primitive_root_of_unity(n), reverse_bits(x_index, n)));
                const E2 eval = combine_initial(q, batch_index, subgroup_x_init);
                old_eval = eadd(emul(old_eval, betas[r]), eval);
                batch_index++;
            }
        }
        if (batch_index != n_instances) return 17;  // "Wrong number of folded instances."
        E2 acc = e2(0);
        for (size_t k = final_poly.size(); k-- > 0;) acc = eadd(escale(acc, subgroup_x), final_poly[k]);
        if (!eeq(acc, old_eval)) return 16;
    }
    return 0;
}

// verify_fri_proof, fri/verifier.rs:62-241 with challenges from challenges.rs:28-75
int glo_verify_fri_proof(const uint64_t* const* initial_caps, const size_t* oracle_num_polys,
                         const size_t* oracle_leaf_width, size_t n_oracles, const glo_fri_batch* batches,
                         size_t n_batches, const uint64_t* opened_values, uint32_t degree_bits,
                         glo_challenger* ch, const glo_fri_params* params, const uint8_t* proof,
                         size_t proof_len) {
    (void)oracle_num_polys;
    size_t pos = 0;
    bool overrun = false;
    auto get_u64 = [&]() -> u64 {
        if (pos + 8 > proof_len) {
            overrun = true;
            return 0;
        }
        u64 v = 0;
        for (int i = 0; i < 8; i++) v |= (u64)proof[pos + i] << (8 * i);
        pos += 8;
        return v;
    };
    auto get_hash = [&]() {
        Hash h;
        for (int i = 0; i < 4; i++) h.e[i] = get_u64();
        return h;
    };
    uint32_t log_N = degree_bits + params->rate_bits;
    size_t N = (size_t)1 << log_N;
    size_t C = (size_t)1 << params->cap_height;
    uint32_t R = params->num_reductions;
    // ---- parse
    std::vector<std::vector<Hash>> caps(R, std::vector<Hash>(C));
    for (uint32_t r = 0; r < R; r++)
        for (size_t c = 0; c < C; c++) caps[r][c] = get_hash();
    struct Query {
        std::vector<std::vector<u64>> init_leaf;
        std::vector<std::vector<Hash>> init_sib;
        std::vector<std::vector<E2>> evals;
        std::vector<std::vector<Hash>> step_sib;
    };
    std::vector<Query> queries(params->num_query_rounds);
    for (auto& q : queries) {
        for (size_t o = 0; o < n_oracles; o++) {
            std::vector<u64> leaf(oracle_leaf_width[o]);
            for (auto& x : leaf) x = get_u64();
            if (pos >= proof_len) return 10;
            size_t len = proof[pos++];
            std::vector<Hash> sib(len);
            for (auto& h : sib) h = get_hash();
            q.init_leaf.push_back(leaf);
            q.init_sib.push_back(sib);
        }
        for (uint32_t r = 0; r < R; r++) {
            size_t arity = (size_t)1 << params->reduction_arity_bits[r];
            std::vector<E2> ev(arity);
            for (auto& e : ev) {
                e.a = get_u64();
                e.b = get_u64();
            }
            if (pos >= proof_len) return 10;
            size_t len = proof[pos++];
            std::vector<Hash> sib(len);
            for (auto& h : sib) h = get_hash();
            q.evals.push_back(ev);
            q.step_sib.push_back(sib);
        }
    }
    uint32_t final_bits = degree_bits;
    for (uint32_t r = 0; r < R; r++) final_bits -= params->reduction_arity_bits[r];
    std::vector<E2> final_poly((size_t)1 << final_bits);
    for (auto& c : final_poly) {
        c.a = get_u64();
        c.b = get_u64();
    }
    u64 pow_witness = get_u64();
    if (overrun || pos != proof_len) return 10;

    // ---- fri_challenges, challenges.rs:28-75
    E2 fri_alpha = get_extension_challenge(ch);
    std::vector<E2> betas;
    for (uint32_t r = 0; r < R; r++) {
        observe_cap(ch, caps[r]);
        betas.push_back(get_extension_challenge(ch));
    }
    for (auto& c : final_poly) observe_ext(ch, c);
    observe_element(ch, pow_witness);
    u64 pow_response = get_challenge(ch);
    std::vector<size_t> indices;
    for (uint32_t q = 0; q < params->num_query_rounds; q++) indices.push_back((size_t)(get_challenge(ch) % N));

    // ---- PoW, verifier.rs:49-60
    {
        uint32_t lz = pow_response == 0 ? 64 : (uint32_t)__builtin_clzll(pow_response);
        if (lz < params->proof_of_work_bits) return 11;
    }
    // ---- PrecomputedReducedOpenings::from_os_and_alpha, verifier.rs:251-261
    std::vector<E2> reduced_openings;
    {
        size_t off = 0;
        for (size_t b = 0; b < n_batches; b++) {
            E2 acc = e2(0);
            for (size_t j = batches[b].num_polys; j-- > 0;)
                acc = eadd(emul(acc, fri_alpha),
                           E2{opened_values[2 * (off + j)], opened_values[2 * (off + j) + 1]});
            off += batches[b].num_polys;
            reduced_openings.push_back(acc);
        }
    }
    u64 omega_N = primitive_root_of_unity(log_N);
    for (size_t qi = 0; qi < queries.size(); qi++) {
        const Query& q = queries[qi];
        size_t x_index = indices[qi];
        // fri_verify_initial_proof, verifier.rs:111-121
        for (size_t o = 0; o < n_oracles; o++) {
            if (q.init_sib[o].size() != log_N - params->cap_height) return 12;
            if (!merkle_verify(q.init_leaf[o].data(), q.init_leaf[o].size(), x_index, q.init_sib[o].data(),
                               q.init_sib[o].size(), (const Hash*)initial_caps[o]))
                return 13;
        }
        u64 subgroup_x = fmul(MULTIPLICATIVE_GROUP_GENERATOR, fexp(omega_N, reverse_bits(x_index, log_N)));
        // fri_combine_initial, verifier.rs:123-166
        E2 sum = e2(0);
        {
            u64 count = 0;
            for (size_t b = 0; b < n_batches; b++) {
                E2 point{batches[b].point[0], batches[b].point[1]};
                E2 red = e2(0);
                for (size_t j = batches[b].num_polys; j-- > 0;) {
                    u64 ev = q.init_leaf[batches[b].oracle_index[j]][batches[b].poly_index[j]];
                    red = eadd(emul(red, fri_alpha), e2(ev));
                    count++;
                }
                E2 numerator = esub(red, reduced_openings[b]);
                E2 denominator = esub(e2(subgroup_x), point);
                sum = emul(eexp(fri_alpha, count), sum);  // alpha.shift(sum)
                count = 0;
                sum = eadd(sum, emul(numerator, einv(denominator)));
            }
        }
        E2 old_eval = sum;
        for (uint32_t r = 0; r < R; r++) {
            uint32_t arity_bits = params->reduction_arity_bits[r];
            size_t arity = (size_t)1 << arity_bits;
            const std::vector<E2>& evals = q.evals[r];
            size_t coset_index = x_index >> arity_bits;
            size_t within = x_index & (arity - 1);
            if (!eeq(evals[within], old_eval)) return 14;
            // compute_evaluation, verifier.rs:22-47 (Lagrange interpolation at beta)
            {
                u64 g = primitive_root_of_unity(arity_bits);
                std::vector<E2> ev = evals;
                {  // reverse_index_bits_in_place(&mut evals)
                    std::vector<u64> flat(2 * arity);
                    for (size_t i = 0; i < arity; i++) {
                        flat[2 * i] = ev[i].a;
                        flat[2 * i + 1] = ev[i].b;
                    }
                    reverse_index_bits_in_place(flat.data(), arity, 2);
                    for (size_t i = 0; i < arity; i++) ev[i] = E2{flat[2 * i], flat[2 * i + 1]};
                }
                size_t rev_within = reverse_bits(within, arity_bits);
                u64 coset_start = fmul(subgroup_x, fexp(g, arity - rev_within));
                std::vector<E2> xs(arity);
                u64 y = 1;
                for (size_t i = 0; i < arity; i++) {
                    xs[i] = e2(fmul(coset_start, y));
                    y = fmul(y, g);
                }
                E2 beta = betas[r];
                // interpolate, field/src/interpolation.rs:31-66
                E2 result;
                bool hit = false;
                for (size_t i = 0; i < arity; i++)
                    if (eeq(xs[i], beta)) {
                        result = ev[i];
                        hit = true;
                    }
                if (!hit) {
                    E2 l_x = e2(1);
                    for (size_t i = 0; i < arity; i++) l_x = emul(l_x, esub(beta, xs[i]));
                    E2 s = e2(0);
                    for (size_t i = 0; i < arity; i++) {
                        E2 w = e2(1);
                        for (size_t j = 0; j < arity; j++)
                            if (j != i) w = emul(w, esub(xs[i], xs[j]));
                        E2 wi = einv(w);
                        s = eadd(s, emul(emul(wi, einv(esub(beta, xs[i]))), ev[i]));
                    }
                    result = emul(l_x, s);
                }
                old_eval = result;
            }
            // verify_merkle_proof_to_cap(flatten(evals), coset_index, cap_i, proof)
            std::vector<u64> flat(2 * arity);
            for (size_t i = 0; i < arity; i++) {
                flat[2 * i] = evals[i].a;
                flat[2 * i + 1] = evals[i].b;
            }
            if (!merkle_verify(flat.data(), flat.size(), coset_index, q.step_sib[r].data(),
                               q.step_sib[r].size(), caps[r].data()))
                return 15;
            for (uint32_t k = 0; k < arity_bits; k++) subgroup_x = fsqr(subgroup_x);
            x_index = coset_index;
        }
        // final_poly.eval(subgroup_x) == old_eval
        E2 acc = e2(0);
        for (size_t k = final_poly.size(); k-- > 0;) acc = eadd(escale(acc, subgroup_x), final_poly[k]);
        if (!eeq(acc, old_eval)) return 16;
    }
    return 0;
}

}  // extern "C"
