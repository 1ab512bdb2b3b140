// div_magic_check.cpp — host check of the narrow path's division by an invariant amount (tests/test_div_magic.py).
//
// Packs every divisor through pack_var32 (the code hqs_classes_set uses), reads the magic number and the shifts back
// out of the record the way fit_count<RT, u32> does, replays the device's four integer instructions in 32-bit host
// arithmetic and compares with n / d.  Divisors: every d < 2^20, every 2^l + delta with |delta| <= 3, and `n_random`
// pseudo-random d < 2^31 (fixed seed).  Numerators per divisor: 0, d - 1, d, floor((2^32 - 1) / d) * d - 1,
// floor((2^32 - 1) / d) * d and 2^32 - 2.  Prints the number of checks and the first failure; exit code 1 on a failure.
#include "../../include/hqsched.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>

typedef uint32_t u32;
typedef uint64_t u64;

#include "../../hyperqueue_b200/csrc/hqs_solver.cuh"

static u64 n_checks = 0, n_fail = 0;

static void check(u32 d) {
    constexpr int RT = 4;
    const u32 r = d & 3;                              // vary the slot: the shift bytes are packed four to a word
    hqs_variant hv;
    memset(&hv, 0, sizeof hv);
    hv.amount[r] = d;
    hv.weight = 10000;
    VarT<RT, u32> dv;
    memset(&dv, 0, sizeof dv);
    const u64 gs[HQS_MAX_RESOURCES] = {1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1};
    if (!pack_var32<RT>(dv, hv, RT, gs) || dv.amount[r] != d || dv.used_mask != (1u << r)) {
        if (!n_fail++) printf("FAIL d=%u: pack_var32 rejected or misplaced the amount\n", d);
        return;
    }
    u32 m;
    memcpy(&m, &dv.rcpf[r], 4);
    const u32 s = (dv.shw[r >> 2] >> ((r & 3) * 8)) & 0xFFu;
    const u64 top = (0xFFFFFFFFull / d) * d;
    const u64 ns[6] = {0, (u64)d - 1, d, top - 1, top, 0xFFFFFFFEull};
    for (u64 n64 : ns) {
        const u32 n = (u32)n64;
        const u32 t = (u32)(((u64)m * n) >> 32);                  // __umulhi
        const u32 q = (t + ((n - t) >> (s & 1u))) >> (s >> 1);
        ++n_checks;
        if (q != n / d) {
            if (!n_fail++) printf("FAIL d=%u n=%u: magic %u shifts %u gives %u, exact %u\n", d, n, m, s, q, n / d);
        }
    }
}

int main(int argc, char** argv) {
    const u64 n_random = argc > 1 ? strtoull(argv[1], nullptr, 10) : 10000000ull;
    for (u32 d = 1; d < (1u << 20); ++d) check(d);
    for (u32 l = 1; l <= 31; ++l)
        for (int delta = -3; delta <= 3; ++delta) {
            const long long d = (1ll << l) + delta;
            if (d >= 1 && d <= (long long)NARROW_LIMIT) check((u32)d);
        }
    u64 x = 0x9E3779B97F4A7C15ull;
    for (u64 i = 0; i < n_random; ++i) {
        x += 0x9E3779B97F4A7C15ull;                                 // splitmix64
        u64 z = x;
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        z ^= z >> 31;
        const u32 d = (u32)(z % NARROW_LIMIT) + 1;                  // 1 .. 2^31 - 1
        check(d);
    }
    printf("checks %llu failures %llu\n", (unsigned long long)n_checks, (unsigned long long)n_fail);
    return n_fail ? 1 : 0;
}
