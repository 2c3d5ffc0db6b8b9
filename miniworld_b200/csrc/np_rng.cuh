// np_rng.cuh -- numpy's Generator(PCG64) stream, draw for draw.
//
// The reference draws every random number through gymnasium's `self.np_random`
// (Generator(PCG64(SeedSequence(seed))), reference miniworld.py:551): placement
// (`choice(n, p)`, `uniform(low[3], high[3])`, `uniform(-pi, pi)`, miniworld.py:865-901),
// texture variants (`integers(0, n)`, opengl.py:133), level choices (pickupobjects.py:64-65)
// and, under domain randomisation, three `uniform` draws per step (miniworld.py:677-680,
// params.py:99-101).  numpy is a third-party dependency of the reference (numpy>=1.22;
// this image: 2.3.5); the algorithms below restate its published PCG64 / Lemire code paths
// (SURVEY.md appendix B) so that resets and domain-rand steps can run on the device and
// still land on the reference's exact stream.  Seeding runs on either side: mwb_seed() uploads
// a 128-bit state / increment the host built, and rng_seed() below restates SeedSequence(seed)
// -> PCG64 for one integer seed, so that a reset can start an env on a chosen seed without a
// host round trip (mwb_enable_episode_seeds).
#pragma once
#include "hd.h"

struct NpRng {
  uint64_t s_hi, s_lo, inc_hi, inc_lo;
  int32_t has32;
  uint32_t cache;
};

// state = state * 0x2360ED051FC65DA44385DF649FCCF645 + inc (mod 2^128), then XSL-RR output
MWB_DEV uint64_t rng_next64(NpRng& r) {
  const uint64_t MH = 0x2360ED051FC65DA4ULL, ML = 0x4385DF649FCCF645ULL;
  uint64_t lo = r.s_lo * ML;
  uint64_t hi = umulhi64(r.s_lo, ML) + r.s_hi * ML + r.s_lo * MH;
  uint64_t lo2 = lo + r.inc_lo;
  hi = hi + r.inc_hi + (lo2 < lo ? 1u : 0u);
  r.s_lo = lo2;
  r.s_hi = hi;
  uint64_t x = hi ^ lo2;
  unsigned rot = (unsigned)(hi >> 58);
  return (x >> rot) | (x << ((64u - rot) & 63u));
}

// low half of a fresh 64-bit draw; the high half is buffered for the next call
MWB_DEV uint32_t rng_next32(NpRng& r) {
  if (r.has32) {
    r.has32 = 0;
    return r.cache;
  }
  uint64_t v = rng_next64(r);
  r.has32 = 1;
  r.cache = (uint32_t)(v >> 32);
  return (uint32_t)v;
}

// Generator.random(): 53-bit mantissa
MWB_DEV double rng_random(NpRng& r) { return (double)(rng_next64(r) >> 11) * (1.0 / 9007199254740992.0); }

// Generator.uniform(lo, hi) given lo and (hi - lo)
MWB_DEV double rng_uniform(NpRng& r, double lo, double range) { return d_add(lo, d_mul(range, rng_random(r))); }

// Generator.integers(0, n) for 1 <= n <= 2^32: Lemire's bounded method on 32-bit draws;
// n == 1 consumes nothing.
MWB_DEV uint32_t rng_integers(NpRng& r, uint32_t n) {
  uint32_t rng = n - 1u;
  if (rng == 0u) return 0u;
  if (rng == 0xFFFFFFFFu) return rng_next32(r);
  uint32_t excl = rng + 1u;
  uint64_t m = (uint64_t)rng_next32(r) * (uint64_t)excl;
  uint32_t left = (uint32_t)m;
  if (left < excl) {
    uint32_t thr = (0xFFFFFFFFu - rng) % excl;
    while (left < thr) {
      m = (uint64_t)rng_next32(r) * (uint64_t)excl;
      left = (uint32_t)m;
    }
  }
  return (uint32_t)(m >> 32);
}

// Generator(PCG64(SeedSequence(seed))) for one integer seed below 2^64: numpy's SeedSequence entropy pool
// (_bit_generator.pyx: mix_entropy, generate_state) and pcg64_srandom_r, in integer arithmetic only.  A seed below 2^32
// is the one-word entropy [seed]; the pool pads missing words with 0, which the zero high word of such a seed already
// is, so both cases read (low word, high word, 0, 0).  include/mwb.h (mwb_enable_episode_seeds) states the algorithm.
MWB_DEV NpRng rng_seed(uint64_t seed) {
  uint32_t hc = 0x43b0d7e5u;
  uint32_t pool[4];
#define MWB_HASHMIX(out, in)   \
  {                            \
    uint32_t v_ = (in) ^ hc;   \
    hc *= 0x931e8875u;         \
    v_ *= hc;                  \
    (out) = v_ ^ (v_ >> 16);   \
  }
  MWB_HASHMIX(pool[0], (uint32_t)seed);
  MWB_HASHMIX(pool[1], (uint32_t)(seed >> 32));
  MWB_HASHMIX(pool[2], 0u);
  MWB_HASHMIX(pool[3], 0u);
#pragma unroll
  for (int src = 0; src < 4; ++src)
#pragma unroll
    for (int dst = 0; dst < 4; ++dst)
      if (src != dst) {
        uint32_t y;
        MWB_HASHMIX(y, pool[src]);
        const uint32_t r = 0xca01f9ddu * pool[dst] - 0x4973f715u * y;
        pool[dst] = r ^ (r >> 16);
      }
#undef MWB_HASHMIX
  // generate_state(4, uint64): eight 32-bit words, paired low word first
  uint32_t w[8];
  hc = 0x8b51f9ddu;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    uint32_t v = pool[k & 3] ^ hc;
    hc *= 0x58f38dedu;
    v *= hc;
    w[k] = v ^ (v >> 16);
  }
  const uint64_t q0 = w[0] | ((uint64_t)w[1] << 32), q1 = w[2] | ((uint64_t)w[3] << 32);
  const uint64_t q2 = w[4] | ((uint64_t)w[5] << 32), q3 = w[6] | ((uint64_t)w[7] << 32);
  // pcg64_srandom_r(initstate = q0 << 64 | q1, initseq = q2 << 64 | q3):
  // inc = initseq << 1 | 1;  state = 0;  step;  state += initstate;  step
  NpRng r;
  r.inc_hi = (q2 << 1) | (q3 >> 63);
  r.inc_lo = (q3 << 1) | 1u;
  r.s_hi = r.s_lo = 0;
  r.has32 = 0;
  r.cache = 0;
  rng_next64(r);
  const uint64_t lo = r.s_lo + q1;
  r.s_hi = r.s_hi + q0 + (lo < r.s_lo ? 1u : 0u);
  r.s_lo = lo;
  rng_next64(r);
  return r;
}
