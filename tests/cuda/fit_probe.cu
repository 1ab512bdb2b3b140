// fit_probe.cu — test probe of the solver's fit count (hyperqueue_b200/csrc/hqs_solver.cuh::fit_count).
//
// Evaluates fit_count<RT, AT> on the GPU for arrays of (free vector, variant, untouched mask, cap) and writes one u64 per
// case.  The variant records are packed by the library's own host helpers (pack_var64 / pack_var32), so the fp32
// reciprocals and the division magic of the narrow path are exercised as hqs_classes_set builds them.  Test
// infrastructure: built next to the oracle's judge library by __graft_entry__.build(), never loaded by the product.
#include "../../include/hqsched.h"

#include <cuda_runtime.h>

#include <cstdio>
#include <cstring>
#include <vector>

namespace {

typedef uint32_t u32;
typedef uint64_t u64;

#include "../../hyperqueue_b200/csrc/hqs_solver.cuh"

template <int RT, typename AT>
__global__ void fit_probe_k(const AT* fr, const VarT<RT, AT>* dv, const u32* untouched, const u64* cap, u64* out, u32 n) {
    const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    AT f[RT];
#pragma unroll
    for (int r = 0; r < RT; ++r) f[r] = fr[(size_t)i * RT + r];
    out[i] = fit_count<RT>(f, untouched[i], dv[i], cap[i]);
}

int fail(char* err, size_t errlen, const char* msg, u64 i = ~0ull) {
    if (err && errlen) {
        if (i == ~0ull) snprintf(err, errlen, "%s", msg);
        else snprintf(err, errlen, "case %llu: %s", (unsigned long long)i, msg);
    }
    return -1;
}

template <typename T>
struct DevBuf {
    T* p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
    cudaError_t alloc(size_t n) { return cudaMalloc(&p, n * sizeof(T)); }
};

template <int RT, typename AT>
int run(u32 n, u32 R, const u64* free_in, const u64* amount, const u32* all_mask, const u64* gscale, const u32* untouched,
        const u64* cap, u64* out, char* err, size_t errlen) {
    constexpr bool NARROW = sizeof(AT) == 4;
    std::vector<AT> fr((size_t)n * RT, 0);
    std::vector<VarT<RT, AT>> dv(n);
    memset(dv.data(), 0, dv.size() * sizeof(VarT<RT, AT>));
    u64 gs[HQS_MAX_RESOURCES];
    for (u32 r = 0; r < HQS_MAX_RESOURCES; ++r) gs[r] = (gscale && r < R) ? gscale[r] : 1;
    for (u32 r = 0; r < R; ++r)
        if (gs[r] == 0) return fail(err, errlen, "gscale must be >= 1");
    for (u32 i = 0; i < n; ++i) {
        if (cap[i] >> 32) return fail(err, errlen, "cap must be below 2^32", i);
        if (all_mask[i] >> R) return fail(err, errlen, "all_mask uses a resource >= R", i);
        hqs_variant hv;
        memset(&hv, 0, sizeof hv);
        hv.all_mask = all_mask[i];
        hv.weight = 10000;
        for (u32 r = 0; r < R; ++r) {
            const u64 a = amount[(size_t)i * R + r], f = free_in[(size_t)i * R + r];
            hv.amount[r] = a;
            if (NARROW && f > 0xFFFFFFFFull) return fail(err, errlen, "narrow free amount above 2^32 - 1", i);
            if (NARROW && a % gs[r]) return fail(err, errlen, "amount is not a multiple of gscale", i);
            fr[(size_t)i * RT + r] = (AT)f;
        }
        bool ok = true;
        if constexpr (NARROW) ok = pack_var32<RT>(dv[i], hv, R, gs);
        else pack_var64<RT>(dv[i], hv, R);
        if (!ok) return fail(err, errlen, "scaled amount above the narrow limit (2^31 - 1)", i);
        if (dv[i].used_mask == 0) return fail(err, errlen, "empty request", i);
    }
    DevBuf<AT> d_fr;
    DevBuf<VarT<RT, AT>> d_dv;
    DevBuf<u32> d_unt;
    DevBuf<u64> d_cap, d_out;
    cudaError_t e = cudaSuccess;
    if (!e) e = d_fr.alloc(fr.size());
    if (!e) e = d_dv.alloc(n);
    if (!e) e = d_unt.alloc(n);
    if (!e) e = d_cap.alloc(n);
    if (!e) e = d_out.alloc(n);
    if (!e) e = cudaMemcpy(d_fr.p, fr.data(), fr.size() * sizeof(AT), cudaMemcpyHostToDevice);
    if (!e) e = cudaMemcpy(d_dv.p, dv.data(), (size_t)n * sizeof(VarT<RT, AT>), cudaMemcpyHostToDevice);
    if (!e) e = cudaMemcpy(d_unt.p, untouched, (size_t)n * 4, cudaMemcpyHostToDevice);
    if (!e) e = cudaMemcpy(d_cap.p, cap, (size_t)n * 8, cudaMemcpyHostToDevice);
    if (!e) {
        fit_probe_k<RT, AT><<<(n + 255) / 256, 256>>>(d_fr.p, d_dv.p, d_unt.p, d_cap.p, d_out.p, n);
        e = cudaGetLastError();
    }
    if (!e) e = cudaMemcpy(out, d_out.p, (size_t)n * 8, cudaMemcpyDeviceToHost);
    if (e) return fail(err, errlen, cudaGetErrorString(e));
    return 0;
}

}  // namespace

// rt: 4, 8 or 16 resource slots; narrow: 0 = u64 amounts, 1 = gcd-scaled u32 amounts (free values are then the scaled
// free amounts themselves, 0xFFFFFFFF = unbounded).  free_rw / amount: [n][R] with R <= rt; all_mask, untouched: [n];
// gscale: [R] or null (all 1); cap: [n], each < 2^32.  Returns 0, or -1 with the reason in err.
extern "C" int hqs_fit_probe(uint32_t rt, int narrow, uint32_t n, uint32_t R, const uint64_t* free_rw, const uint64_t* amount,
                             const uint32_t* all_mask, const uint64_t* gscale, const uint32_t* untouched, const uint64_t* cap,
                             uint64_t* out, char* err, size_t errlen) {
    if (err && errlen) err[0] = 0;
    if (rt != 4 && rt != 8 && rt != 16) return fail(err, errlen, "rt must be 4, 8 or 16");
    if (R == 0 || R > rt) return fail(err, errlen, "R must be in 1..rt");
    if (n == 0) return 0;
    if (n > (1u << 24)) return fail(err, errlen, "at most 2^24 cases per call");
    if (!free_rw || !amount || !all_mask || !untouched || !cap || !out) return fail(err, errlen, "null array");
    if (narrow) {
        if (rt == 4) return run<4, u32>(n, R, free_rw, amount, all_mask, gscale, untouched, cap, out, err, errlen);
        if (rt == 8) return run<8, u32>(n, R, free_rw, amount, all_mask, gscale, untouched, cap, out, err, errlen);
        return run<16, u32>(n, R, free_rw, amount, all_mask, gscale, untouched, cap, out, err, errlen);
    }
    if (rt == 4) return run<4, u64>(n, R, free_rw, amount, all_mask, gscale, untouched, cap, out, err, errlen);
    if (rt == 8) return run<8, u64>(n, R, free_rw, amount, all_mask, gscale, untouched, cap, out, err, errlen);
    return run<16, u64>(n, R, free_rw, amount, all_mask, gscale, untouched, cap, out, err, errlen);
}
