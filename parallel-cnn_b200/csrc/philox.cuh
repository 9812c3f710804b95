// parallel-cnn_b200/csrc/philox.cuh -- Philox4x32-10, the counter-based generator behind every random draw of the library
// (dropout.cu's masks, augment.cu's permutation and crops).  A draw is a pure function of (counter, key), so the bits depend on
// neither the launch grid nor the GPU, and tests/dropout_ref.py replays them in numpy.
#pragma once

// Philox4x32-10 (Salmon et al., SC'11; Random123): ten rounds of two 32x32->64 multiplies, the key bumped by the Weyl constants
// between rounds
__device__ __forceinline__ uint4 philox4x32_10(unsigned c0, unsigned c1, unsigned c2, unsigned c3, unsigned k0, unsigned k1) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        const unsigned lo0 = 0xD2511F53u * c0, hi0 = __umulhi(0xD2511F53u, c0);
        const unsigned lo1 = 0xCD9E8D57u * c2, hi1 = __umulhi(0xCD9E8D57u, c2);
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return make_uint4(c0, c1, c2, c3);
}
