// rng.cuh -- per-path Philox4x32-10 stream and the rand 0.8 / rand_distr 0.4
// distributions the reference draws from (SURVEY 8a-RNG):
//   gen::<f64>()      src/material.rs:247, src/shape/mesh.rs:85-90, src/shape/cube.rs:75-76
//   gen_range(a..b)   src/renderer.rs:137-138
//   gen_bool(p)       src/material.rs:264
//   Uniform(0..n)     src/kdtree.rs:140, src/shape/cube.rs:77
//   UnitDisc          src/camera.rs:73, src/shape/sphere.rs:53, src/material.rs:271
//   UnitCircle        src/material.rs:251
// The reference seeds ChaCha12 from OS entropy per row (src/renderer.rs:121); here
// key = (seed_lo, seed_hi), counter = (block, pixel, sample_lo, sample_hi).
// A path's stream of 64-bit draws is TWO Philox streams side by side: draw 4b + w has word w of block b as its high
// half and word w of block (b | 2^31) as its low half.  The f32 kernels only ever look at the high half of a draw (24
// bits of it make a float), so they compute the first stream alone and use all four words of every block; the f64
// gate and the oracle compute both.  (Until round 2 a block was cut into two 64-bit draws and the f32 path threw the
// low words away: half of its Philox work -- a quarter of Cornell's warp instructions, ncu -- bought nothing.)
constexpr uint32_t PHILOX_LOW_STREAM = 0x80000000u;
#pragma once
#include "vec.cuh"

namespace rptb {

struct Philox {
    uint32_t key0, key1;
    uint32_t block, pixel, samp_lo, samp_hi;
    uint64_t d1, d2, d3;  // the draws of the current block pair not handed out yet, next first
    uint32_t left;

    RPTB_HD void init(uint64_t seed, uint32_t pix, uint64_t sample) {
        key0 = (uint32_t)seed;
        key1 = (uint32_t)(seed >> 32);
        block = 0;
        pixel = pix;
        samp_lo = (uint32_t)sample;
        samp_hi = (uint32_t)(sample >> 32);
        left = 0;
        d1 = d2 = d3 = 0;
    }

    static RPTB_HD void mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo) {
#ifdef __CUDA_ARCH__
        lo = a * b;
        hi = __umulhi(a, b);
#else
        const uint64_t p = (uint64_t)a * b;
        lo = (uint32_t)p;
        hi = (uint32_t)(p >> 32);
#endif
    }

    static RPTB_HD void block10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1,
                                uint32_t out[4]) {
#pragma unroll
        for (int i = 0; i < 10; i++) {
            uint32_t hi0, lo0, hi1, lo1;
            mulhilo(0xD2511F53u, c0, hi0, lo0);
            mulhilo(0xCD9E8D57u, c2, hi1, lo1);
            const uint32_t n0 = hi1 ^ c1 ^ k0;
            const uint32_t n2 = hi0 ^ c3 ^ k1;
            c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
            k0 += 0x9E3779B9u;
            k1 += 0xBB67AE85u;
        }
        out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
    }

    // One Philox block costs ~60 instructions; the integrator draws from ~20 call sites, so
    // the block function is kept out of line (a pure function of register arguments: one
    // copy in the instruction cache instead of 20, generator state stays in registers).
#ifdef __CUDA_ARCH__
    static __device__ __noinline__ uint4 block_call(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                    uint32_t k1) {
        uint32_t o[4];
        block10(c0, c1, c2, c3, k0, k1, o);
        return make_uint4(o[0], o[1], o[2], o[3]);
    }
#endif
    RPTB_HD uint64_t refill() {
#ifdef __CUDA_ARCH__
        const uint4 vh = block_call(block, pixel, samp_lo, samp_hi, key0, key1);
        const uint4 vl = block_call(block | PHILOX_LOW_STREAM, pixel, samp_lo, samp_hi, key0, key1);
        const uint32_t hi[4] = {vh.x, vh.y, vh.z, vh.w}, lo[4] = {vl.x, vl.y, vl.z, vl.w};
#else
        uint32_t hi[4], lo[4];
        block10(block, pixel, samp_lo, samp_hi, key0, key1, hi);
        block10(block | PHILOX_LOW_STREAM, pixel, samp_lo, samp_hi, key0, key1, lo);
#endif
        block++;
        d1 = ((uint64_t)hi[1] << 32) | lo[1];
        d2 = ((uint64_t)hi[2] << 32) | lo[2];
        d3 = ((uint64_t)hi[3] << 32) | lo[3];
        left = 3;
        return ((uint64_t)hi[0] << 32) | lo[0];
    }

    RPTB_HD uint64_t next_u64() {
        if (left == 0) return refill();
        const uint64_t v = d1;
        d1 = d2;
        d2 = d3;
        left--;
        return v;
    }
};

template <class R>
struct Rng;

// f64: bit-for-bit the oracle's conversions of the 64-bit draws.
template <>
struct Rng<double> {
    Philox p;
    RPTB_HD void init(uint64_t seed, uint32_t pix, uint64_t sample) { p.init(seed, pix, sample); }
    RPTB_HD void bind(uint32_t*, uint32_t) {}
    RPTB_HD void ensure() {}
    template <class W>
    RPTB_HD void ensure(unsigned, uint32_t) {}
    RPTB_HD double gen() { return (double)(p.next_u64() >> 11) * (1.0 / 9007199254740992.0); }
    RPTB_HD double u52() { return (double)(p.next_u64() >> 12) * (1.0 / 4503599627370496.0); }
    // Rng::gen_bool(p): Bernoulli -> u64 < p * 2^64
    RPTB_HD bool bernoulli(double prob) {
        const uint64_t v = p.next_u64();
        if (prob >= 1.0) return true;
        return v < (uint64_t)(prob * 18446744073709551616.0);
    }
    // Rng::gen::<bool>(): the top bit of one draw
    RPTB_HD bool coin() { return (p.next_u64() >> 63) != 0; }
    // Uniform::from(0..n) for usize: widening multiply with rejection zone
    RPTB_HD uint64_t below(uint64_t n) {
        const uint64_t ints_to_reject = (0xFFFFFFFFFFFFFFFFull - n + 1) % n;
        const uint64_t zone = 0xFFFFFFFFFFFFFFFFull - ints_to_reject;
        while (true) {
            const uint64_t v = p.next_u64();
            const uint64_t lo = v * n;
#ifdef __CUDA_ARCH__
            const uint64_t hi = __umul64hi(v, n);
#else
            const uint64_t hi = (uint64_t)(((unsigned __int128)v * n) >> 64);
#endif
            if (lo <= zone) return hi;
        }
    }
};

// f32: only the HIGH 32-bit word of each 64-bit draw is kept -- its top 24 bits are the f64
// value truncated to a float in [0,1), so both precisions see the same stream -- and the high
// words are the first Philox stream's words in order (see the top of the file): a block is four
// draws.  They wait in a register FIFO (RngBuf below) that ensure() refills -- the integrator
// calls it where the whole warp is converged: the ~60-instruction Philox block then runs once
// for 32 lanes instead of once per lane per call site (`half` counts pairs of draws produced).
// gen_bool / Uniform(0..n) decide on the high word alone; the decision differs from the
// 64-bit one with probability <= n * 2^-32 per draw (f32 mode only).
// How the four draws of a block are buffered is a template parameter (same stream, bit for bit, whichever):
//   BUF_PAIR  two draws enter a 4-entry FIFO, the other two wait in s0/s1           (6 words)
//   BUF_FOUR  a 4-entry FIFO, refilled when empty                                    (4 words)
//   BUF_EIGHT an 8-entry FIFO; a block enters whenever four entries are free          (8 words)
// No one of them was fastest on every scene when they were compared (before the port to the H100; not re-measured
// there).  (Two more were tried and dropped -- the current block in a 4-entry FIFO plus the whole next block beside it,
// handed over at the draw that empties the FIFO or at the next draw after, and the shared-memory ring below: neither
// beat EIGHT.)
// EIGHT keeps ensure() -- the converged point -- the place where nearly every block is computed (a lane holds >= 4
// draws after it, and few slots draw more); FOUR is the smallest in registers, which is what the 64-register kernels of
// the mesh scenes (F_BVH, 8 CTAs per SM) want.  The megakernel picks per instantiation (integrator.cuh, MegaRng).
enum { BUF_PAIR = 0, BUF_FOUR = 1, BUF_EIGHT = 2 };
#ifndef RPTB_FIFO_MODE
#define RPTB_FIFO_MODE 2      // Rng<float>, and the megakernel's generator for scenes without a BVH
#endif
#ifndef RPTB_FIFO_MODE_BVH
#define RPTB_FIFO_MODE_BVH 1  // the megakernel's generator in F_BVH instantiations
#endif

template <int BUF>
struct RngBuf;  // state + push_block() / ensure() / next32() / save() / load()

struct RngStream {  // which block comes next
    uint32_t key0, key1, half, pixel, samp_lo, samp_hi;  // half: pairs of draws produced so far (block = half >> 1)
    RPTB_HD void init_stream(uint64_t seed, uint32_t pix, uint64_t sample) {
        key0 = (uint32_t)seed;
        key1 = (uint32_t)(seed >> 32);
        half = 0;
        pixel = pix;
        samp_lo = (uint32_t)sample;
        samp_hi = (uint32_t)(sample >> 32);
    }
    RPTB_HD void block4(uint32_t o[4]) {
#ifdef __CUDA_ARCH__
        const uint4 v = Philox::block_call(half >> 1, pixel, samp_lo, samp_hi, key0, key1);
        o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
#else
        Philox::block10(half >> 1, pixel, samp_lo, samp_hi, key0, key1, o);
#endif
    }
};

template <>
struct RngBuf<BUF_PAIR> : RngStream {
    uint32_t q0, q1, q2, q3, s0, s1, avail;
    RPTB_HD void clear() { q0 = q1 = q2 = q3 = s0 = s1 = 0; avail = 0; }
    RPTB_HD void save(uint32_t* w) const { w[0] = q0; w[1] = q1; w[2] = q2; w[3] = q3; w[4] = s0; w[5] = s1; }
    RPTB_HD void load(const uint32_t* w) { q0 = w[0]; q1 = w[1]; q2 = w[2]; q3 = w[3]; s0 = w[4]; s1 = w[5]; }
    RPTB_HD void push_block() {  // the next two draws of the stream; requires avail <= 2
        uint32_t a, b;
        if (half & 1u) {
            a = s0;
            b = s1;
        } else {
            uint32_t o[4];
            block4(o);
            a = o[0]; b = o[1]; s0 = o[2]; s1 = o[3];
        }
        half++;
        if (avail == 0) { q0 = a; q1 = b; }
        else if (avail == 1) { q1 = a; q2 = b; }
        else { q2 = a; q3 = b; }
        avail += 2;
    }
    RPTB_HD void ensure() {
        if (avail <= 2) push_block();
        if (avail <= 2) push_block();
    }
    RPTB_HD uint32_t next32() {
        if (avail == 0) push_block();  // a slot consumed more than the FIFO held
        const uint32_t v = q0;
        q0 = q1; q1 = q2; q2 = q3;
        avail--;
        return v;
    }
};

template <>
struct RngBuf<BUF_FOUR> : RngStream {
    uint32_t q0, q1, q2, q3, avail;
    RPTB_HD void clear() { q0 = q1 = q2 = q3 = 0; avail = 0; }
    RPTB_HD void save(uint32_t* w) const { w[0] = q0; w[1] = q1; w[2] = q2; w[3] = q3; }
    RPTB_HD void load(const uint32_t* w) { q0 = w[0]; q1 = w[1]; q2 = w[2]; q3 = w[3]; }
    RPTB_HD void push_block() {  // a whole block; requires avail == 0
        uint32_t o[4];
        block4(o);
        half += 2;
        q0 = o[0]; q1 = o[1]; q2 = o[2]; q3 = o[3];
        avail = 4;
    }
    RPTB_HD void ensure() {
        if (avail == 0) push_block();
    }
    RPTB_HD uint32_t next32() {
        if (avail == 0) push_block();
        const uint32_t v = q0;
        q0 = q1; q1 = q2; q2 = q3;
        avail--;
        return v;
    }
};

template <>
struct RngBuf<BUF_EIGHT> : RngStream {
    uint32_t q0, q1, q2, q3, q4, q5, q6, q7, avail;
    RPTB_HD void clear() { q0 = q1 = q2 = q3 = q4 = q5 = q6 = q7 = 0; avail = 0; }
    RPTB_HD void save(uint32_t* w) const { w[0] = q0; w[1] = q1; w[2] = q2; w[3] = q3; w[4] = q4; w[5] = q5; w[6] = q6; w[7] = q7; }
    RPTB_HD void load(const uint32_t* w) { q0 = w[0]; q1 = w[1]; q2 = w[2]; q3 = w[3]; q4 = w[4]; q5 = w[5]; q6 = w[6]; q7 = w[7]; }
    RPTB_HD void push_block() {  // a whole block; requires avail <= 4
        uint32_t o[4];
        block4(o);
        half += 2;
        switch (avail) {
            case 0: q0 = o[0]; q1 = o[1]; q2 = o[2]; q3 = o[3]; break;
            case 1: q1 = o[0]; q2 = o[1]; q3 = o[2]; q4 = o[3]; break;
            case 2: q2 = o[0]; q3 = o[1]; q4 = o[2]; q5 = o[3]; break;
            case 3: q3 = o[0]; q4 = o[1]; q5 = o[2]; q6 = o[3]; break;
            default: q4 = o[0]; q5 = o[1]; q6 = o[2]; q7 = o[3]; break;
        }
        avail += 4;
    }
    RPTB_HD void ensure() {
        if (avail <= 4) push_block();
    }
    // the refill at a draw site (a slot drew more than the FIFO held): the FIFO is empty, so no placement by count --
    // next32() is inlined at ~20 sites, and with the switch above at each of them the kernel outgrew the instruction
    // cache (ncu, Cornell: stall no_instruction 0.57 -> 2.58 warps per issue, issue-active 70.6 -> 65.6 %)
    RPTB_HD void refill_empty() {
        uint32_t o[4];
        block4(o);
        half += 2;
        q0 = o[0]; q1 = o[1]; q2 = o[2]; q3 = o[3];
        avail = 4;
    }
    RPTB_HD uint32_t next32() {
        if (avail == 0) refill_empty();
        const uint32_t v = q0;
        q0 = q1; q1 = q2; q2 = q3; q3 = q4; q4 = q5; q5 = q6; q6 = q7;
        avail--;
        return v;
    }
};

template <int BUF>
struct RngF32 : RngBuf<BUF> {
    static constexpr int STATE_WORDS = 8;  // what save() may write
    RPTB_HD void init(uint64_t seed, uint32_t pix, uint64_t sample) {
        this->init_stream(seed, pix, sample);
        this->clear();
    }
    template <class W>
    RPTB_HD void ensure(unsigned, uint32_t) { RngBuf<BUF>::ensure(); }  // (topping up to the slot's expected draws instead was measured too, and was slower)
    RPTB_HD void ensure() { RngBuf<BUF>::ensure(); }
    RPTB_HD void bind(uint32_t*, uint32_t) {}
    RPTB_HD float gen() { return (float)(this->next32() >> 8) * (1.0f / 16777216.0f); }
    RPTB_HD float u52() { return gen(); }
    RPTB_HD bool bernoulli(float prob) {
        const uint32_t v = this->next32();
        if (prob >= 1.0f) return true;
        return v < (uint32_t)((uint64_t)((double)prob * 18446744073709551616.0) >> 32);
    }
    RPTB_HD bool coin() { return (this->next32() >> 31) != 0; }
    RPTB_HD uint64_t below(uint64_t n) {
#ifdef __CUDA_ARCH__
        return (uint64_t)__umulhi(this->next32(), (uint32_t)n);
#else
        return ((uint64_t)this->next32() * (uint32_t)n) >> 32;
#endif
    }
};
template <>
struct Rng<float> : RngF32<RPTB_FIFO_MODE> {};

// The alternative to the register FIFOs (RPTB_RNG_FIFO 0; what the vertex-at-once engine draws from): the same stream
// as Rng<float> (high word of every 64-bit draw), buffered in an
// 8-entry ring per thread that lives in SHARED memory on the device (entry i of thread t at ring[i * stride + t]:
// one bank per lane, no conflicts; a ring in registers would need shuffling moves per draw and four more live
// registers in a kernel that already spills).  What this buys: with the 4-entry register FIFO a slot that drew more
// than the FIFO held refilled it inside whatever rejection loop it was in -- the ~60-instruction Philox block ran on a
// few lanes of the warp at a time.  ensure() tops a lane up to
// what it is about to draw where the warp is converged, and all lanes that need a block compute it together.
constexpr uint32_t RNG_RING = 8;
#ifndef RPTB_RNG_FILL
#define RPTB_RNG_FILL 0
#endif
#ifndef RPTB_RNG_FIFO
// 1 = the slot engine keeps a register FIFO (RngF32), 0 = it draws from the ring below.  The ring raises the lanes per
// Philox instruction, but its shared-memory traffic and vote loops cost more than that saves (measured with everything
// else equal, before the port to the H100), so the FIFO is the default and the ring is what the vertex-at-once engine
// (integrator_vx.cuh) uses.
#define RPTB_RNG_FIFO 1
#endif
struct RngRing {
    uint32_t key0, key1, block, pixel, samp_lo, samp_hi;
    uint32_t head, avail;
    uint32_t* ring;     // device: shared memory; host emulation: `own`
    uint32_t stride;
#ifdef __CUDA_ARCH__
    // (a local object of device code only: it never crosses the host/device boundary, so the layouts may differ)
    __device__ void bind(uint32_t* shared_ring, uint32_t shared_stride) { ring = shared_ring; stride = shared_stride; }
#else
    uint32_t own[RNG_RING];
    void bind(uint32_t* shared_ring, uint32_t shared_stride) {
        if (shared_ring) { ring = shared_ring; stride = shared_stride; }
        else { ring = own; stride = 1; }
    }
#endif
    RPTB_HD void init(uint64_t seed, uint32_t pix, uint64_t sample) {
        key0 = (uint32_t)seed;
        key1 = (uint32_t)(seed >> 32);
        block = 0;
        pixel = pix;
        samp_lo = (uint32_t)sample;
        samp_hi = (uint32_t)(sample >> 32);
        head = 0;
        avail = 0;
    }
    RPTB_HD uint32_t& at(uint32_t i) { return ring[(i & (RNG_RING - 1u)) * stride]; }
    RPTB_HD void push_block() {  // four draws; requires avail <= RNG_RING - 4
#ifdef __CUDA_ARCH__
        const uint4 v = Philox::block_call(block, pixel, samp_lo, samp_hi, key0, key1);
        const uint32_t o[4] = {v.x, v.y, v.z, v.w};
#else
        uint32_t o[4];
        Philox::block10(block, pixel, samp_lo, samp_hi, key0, key1, o);
#endif
        block++;
        at(head + avail) = o[0];
        at(head + avail + 1u) = o[1];
        at(head + avail + 2u) = o[2];
        at(head + avail + 3u) = o[3];
        avail += 4;
    }
    // W = the warp policy of integrator.cuh (real votes on the device, a single lane in host emulation).  `need` = how
    // many draws this lane expects to take before the next converged point (0 for a lane that will draw nothing): the
    // lanes that are short compute their blocks together, nobody generates draws on speculation -- a path that ends
    // after two draws (a camera ray that leaves the scene) costs one Philox block, not a ring full.
    template <class W>
    RPTB_HD void ensure(unsigned mask, uint32_t need) {
        // (a block is four entries: a lane can take one while avail <= RNG_RING - 4)
#if RPTB_RNG_FILL
        // A/B switch: top every lane up to >= 6 entries whatever it is about to draw
        (void)need;
        while (W::any(mask, avail <= RNG_RING - 4u)) {
            if (avail <= RNG_RING - 4u) push_block();
        }
#else
        while (W::any(mask, avail < need && avail <= RNG_RING - 4u)) {
            if (avail < need && avail <= RNG_RING - 4u) push_block();
        }
#endif
    }
    RPTB_HD uint32_t next32() {
        if (avail == 0) push_block();  // a slot consumed more than the ring held
        const uint32_t v = at(head);
        head++;
        avail--;
        return v;
    }
    RPTB_HD float gen() { return (float)(next32() >> 8) * (1.0f / 16777216.0f); }
    RPTB_HD float u52() { return gen(); }
    RPTB_HD bool bernoulli(float prob) {
        const uint32_t v = next32();
        if (prob >= 1.0f) return true;
        return v < (uint32_t)((uint64_t)((double)prob * 18446744073709551616.0) >> 32);
    }
    RPTB_HD bool coin() { return (next32() >> 31) != 0; }
    RPTB_HD uint64_t below(uint64_t n) {
#ifdef __CUDA_ARCH__
        return (uint64_t)__umulhi(next32(), (uint32_t)n);
#else
        return ((uint64_t)next32() * (uint32_t)n) >> 32;
#endif
    }
};

// Rng::gen_range(lo..hi) -> UniformFloat::sample_single
template <class R, class RNG>
RPTB_HD R gen_range(RNG& r, R lo, R hi) {
    const R scale = hi - lo;
    while (true) {
        const R v12 = (R)1 + r.u52();
        const R res = v12 * scale + (lo - scale);
        if (res < hi) return res;
    }
}
// Uniform::new(-1, 1).sample
template <class R, class RNG>
RPTB_HD R uniform_pm1(RNG& r) { return r.u52() * (R)2 + (R)(-1); }

// Rng::gen_bool(p).  p >= 1 returns true (the reference's ALWAYS_TRUE case) but still
// consumes one draw so that the number of draws per vertex is material-independent.
template <class R, class RNG>
RPTB_HD bool gen_bool(RNG& r, R prob) { return r.bernoulli(prob); }

// Uniform::from(0..n) for usize
template <class RNG>
RPTB_HD uint64_t uniform_usize(RNG& r, uint64_t n) { return r.below(n); }

// rand_distr::UnitDisc: rejection from the square, boundary inclusive
template <class R, class RNG>
RPTB_HD void unit_disc(RNG& r, R& x, R& y) {
    while (true) {
        x = uniform_pm1<R>(r);
        y = uniform_pm1<R>(r);
        if (x * x + y * y <= (R)1) return;
    }
}
// rand_distr::UnitCircle: von Neumann's method
template <class R, class RNG>
RPTB_HD void unit_circle(RNG& r, R& x, R& y) {
    R x1, x2, sum;
    while (true) {
        x1 = uniform_pm1<R>(r);
        x2 = uniform_pm1<R>(r);
        sum = x1 * x1 + x2 * x2;
        if (sum < (R)1) break;
    }
    const R diff = x1 * x1 - x2 * x2;
    x = diff / sum;
    y = (R)2 * x1 * x2 / sum;
}

}  // namespace rptb
