// Eight SHAKE128 sponges advancing in lock step on one core: Keccak-f[1600] on 8 independent states held lane-interleaved
// in 25 zmm registers (AVX-512F: vprolq for rho, vpternlogq for theta's three-way xor and for chi).  One sponge is
// strictly sequential, but a PRSS call squeezes C(m-1, t) of them -- one per key subset (thresha.py:257) -- and when
// the host has fewer cores than subsets (20 subsets for m = 7, t = 3 on an 8-vCPU host) each worker
// thread owns several: x8 squeezes them together.
// All sponges of a group absorb messages of the SAME length (key || uci) and are squeezed by the same amounts.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace mpyc_shake {

bool x8_available();   // AVX-512F present (cpuid) and not disabled by MPYC_B200_NO_AVX512

struct Shake128x8 {
    static constexpr size_t RATE = 168;
    alignas(64) uint64_t st[25][8];   // st[lane][sponge]
    size_t pos;
    bool squeezing;
    int count;                         // active sponges (1..8); the others stay all-zero states

    void reset(int n);
    // absorb len bytes into every active sponge: in[s] points at sponge s's bytes
    void absorb(const uint8_t* const* in, size_t len);
    // squeeze len bytes from every active sponge to out[s]
    void squeeze(uint8_t* const* out, size_t len);

private:
    void finish();
};

}   // namespace mpyc_shake
