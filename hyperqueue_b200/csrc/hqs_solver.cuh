// hqs_solver.cuh — device-side building blocks of the tick: the class table layout, the exact fit count
// (how many tasks of a request fit into a free vector), the pack step (one warp fills one worker) and the
// acquire/release helpers, and the host code that packs a variant into its device record.  Included by hqsched.cu inside
// its anonymous namespace (and by the fit-count probe of the tests); the tick kernel itself is hqs_tick.cuh.
#pragma once

constexpr u32 PACK_MAX_CAND = 64;    // (class, variant) candidates of the packed level: 2 per lane
constexpr u32 PACK_MAX_ITER = 64;
constexpr u32 PACK_CHUNK_DIV = 8;
constexpr u32 HQS_MAX_PEERS = 16;      // ranks of a sharded ready set
constexpr long long SPIN_TIMEOUT_CYCLES = 2000000000ll;   // ~1 s: a stuck grid must not hang the GPU
constexpr long long PEER_TIMEOUT_CYCLES = 30000000000ll;  // ~15 s: another PROCESS may be late by a first-launch module load or an allocation

// Amounts come in two widths.  u64: the ABI's fixed-point fractions as they are.  u32 ("narrow"): the same
// amounts divided by the per-resource gcd of all requested amounts — fit counts are unchanged by that
// (floor(n / d) == floor(floor(n / g) / (d / g)) when g divides d), a quotient is four integer instructions (division
// by an invariant amount, see fit_count) instead of a 64-bit sequence, and the solver's sequential critical path
// shrinks accordingly.  The narrow path is taken when every scaled amount of the tick is below 2^31.
template <int RT, typename AT = u64>
struct VarT {
    AT amount[RT];
    float rcpf[2 * RT];  // [0, RT): u64 amounts: fp32 1.0 / amount (0 where unused); u32 amounts: the BITS of the division
                         // magic (see fit_count); [RT, 2 RT): fp32 of the exact amount
    u64 min_time_ms;
    u32 all_mask;
    u32 used_mask;
    u32 shw[(RT + 3) / 4];   // u32 amounts: one byte per resource, sh1 | sh2 << 1 of the division by the invariant amount
    u32 pad_[((RT + 3) / 4) & 1];
};
template <int RT, typename AT = u64>
struct ClassT {
    u32 n_variants;
    u32 pad;
    VarT<RT, AT> v[HQS_MAX_VARIANTS];
};
template <typename AT> struct AmountMax;
template <> struct AmountMax<u64> { static constexpr u64 value = HQS_AMOUNT_MAX; };
template <> struct AmountMax<u32> { static constexpr u32 value = 0xFFFFFFFFu; };
constexpr u64 NARROW_LIMIT = 0x7FFFFFFFull;      // scaled amounts of the narrow path stay below 2^31

// ---- host: one ABI variant -> its device record (hqs_classes_set; the fit-count probe of the tests uses the same code).
// The caller has checked that the variant requests no resource >= R.
template <int RT>
inline void pack_var64(VarT<RT, u64>& dv, const hqs_variant& hv, u32 R) {
    u32 used = 0;
    for (u32 r = 0; r < R; ++r) {
        const bool all = (hv.all_mask >> r) & 1;
        const u64 amt = hv.amount[r];
        dv.amount[r] = all ? 0 : amt;
        dv.rcpf[r] = (!all && amt) ? 1.0f / (float)amt : 0.0f;
        dv.rcpf[RT + r] = all ? 0.0f : (float)(double)amt;          // u64 -> double -> float, both RN
        if (all || amt) used |= 1u << r;
    }
    dv.min_time_ms = hv.min_time_ms;
    dv.all_mask = hv.all_mask & ((1u << R) - 1);
    dv.used_mask = used;
}

// Magic number and shifts of the division by the invariant amount 1 <= d < 2^32 (see fit_count):
// l = ceil(log2 d), m = floor(2^32 (2^l - d) / d) + 1, sh = min(l, 1) | max(l - 1, 0) << 1.
inline void div_magic(u32 d, u32* magic, u32* sh) {
    u32 l = 0;
    while (l < 32 && ((u64)1 << l) < d) ++l;
    *magic = (u32)((((u64)1 << 32) * (((u64)1 << l) - d)) / d + 1);
    *sh = (l < 1 ? l : 1) | ((l > 0 ? l - 1 : 0) << 1);
}

// The narrow record: amounts divided by the per-resource gcd `gscale` (which divides every requested amount).  Returns
// false if a scaled amount does not fit the narrow path (> NARROW_LIMIT); the record is then not usable.
template <int RT>
inline bool pack_var32(VarT<RT, u32>& dv, const hqs_variant& hv, u32 R, const u64* gscale) {
    bool ok = true;
    u32 used = 0;
    unsigned char* shb = reinterpret_cast<unsigned char*>(dv.shw);         // one byte per resource
    for (u32 r = 0; r < R; ++r) {
        const bool all = (hv.all_mask >> r) & 1;
        const u64 amt = all ? 0 : hv.amount[r] / gscale[r];
        if (amt > NARROW_LIMIT) ok = false;
        dv.amount[r] = (u32)amt;
        if (amt && amt <= NARROW_LIMIT) {
            u32 magic, sh;
            div_magic((u32)amt, &magic, &sh);
            memcpy(&dv.rcpf[r], &magic, 4);
            shb[r] = (unsigned char)sh;
        } else {
            dv.rcpf[r] = 0.0f;
        }
        dv.rcpf[RT + r] = all ? 0.0f : (float)(double)hv.amount[r];
        if (all || hv.amount[r]) used |= 1u << r;
    }
    dv.min_time_ms = hv.min_time_ms;
    dv.all_mask = hv.all_mask & ((1u << R) - 1);
    dv.used_mask = used;
    return ok;
}

#ifdef __CUDACC__
// ---- device side (everything below; a host-only compiler sees the layouts and the packing helpers above)

struct PackScratch {          // global memory, written by the solver CTA, read by the pack warps (and back)
    u64* fr;                  // [W][R]
    u32* quota;               // [W][PACK_MAX_CAND]   per (worker, group of the level)
    u32* taken;               // [W][PACK_MAX_CAND]   per (worker, candidate)
    u32* cand;                // [PACK_MAX_CAND]      class | variant << 16 | group-in-level << 24
    u32* meta;                // [2] n_cand, n_groups
};

__device__ __forceinline__ u32 ld_acquire(const u32* p) {
    u32 v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(u32* p, u32 v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ u32 ld_acquire_sys(const u32* p) {
    u32 v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(u32* p, u32 v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ u64 sat_add64(u64 a, u64 b) {
    const u64 s = a + b;
    return s < a ? HQS_AMOUNT_MAX : s;              // MAX absorbs
}
__device__ __forceinline__ u64 sat_mul64(u64 a, u64 b) {
    return __umul64hi(a, b) ? HQS_AMOUNT_MAX : a * b;
}

template <int RT, typename AT>
__device__ __forceinline__ bool admissible(const VarT<RT, AT>& dv, u32 v, uint8_t blk, u64 rem_time) {
    return !((blk >> v) & 1) && (rem_time == HQS_TIME_INF || dv.min_time_ms <= rem_time);
}

// How many tasks of the variant fit into `fr` now, at most `cap` (< 2^32): min over the requested resources
// of floor(free / amount) (workerload.rs:121-145 without the 1024 cap).  `All`: feasible with >= 1 fraction
// (request.rs:34-36) but consumes the total (solver.rs:120-124), so at most one task and only on an untouched
// resource: bit r of `untouched` says "total[r] != 0 and free[r] == total[r]" (exact amounts).
// This sits on the solver's sequential critical path once per step, so it is STRAIGHT-LINE code: per resource
// (independent => ILP) a multiply-compare "does cap * amount fit" test and an fp32 quotient estimate with an
// exact integer fix-up, combined by selects.  Only a binding quotient of 2^20 or more (one worker taking over
// a million tasks of one group) falls back to an integer division.
template <int RT>
__device__ __forceinline__ u64 fit_count(const u64 (&fr)[RT], u32 untouched, const VarT<RT, u64>& dv, u64 cap) {
    u64 cnt = cap;
    bool big = false;
    const u32 used = dv.used_mask, allm = dv.all_mask;
#pragma unroll
    for (int r = 0; r < RT; ++r) {
        const bool on = (used >> r) & 1, all = (allm >> r) & 1;
        const u64 n = fr[r], d = dv.amount[r];
        const bool fits_cap = __umul64hi(d, cap) == 0 && d * cap <= n;
        // the 64-bit free amount is converted through its 32-bit halves (fp64 and 64-bit divisions cost hundreds of cycles)
        const float nf = __fmaf_rn(__uint2float_rn((u32)(n >> 32)), 4294967296.0f, __uint2float_rn((u32)n));
        const float qf = nf * dv.rcpf[r];
        // the fix-ups compare the full 128-bit product: near 2^64 the estimate can be 2^64 / d (nf rounds up to 2^64),
        // q * d then wraps, and a wrapped product would read as "fits" and over-count
        u64 q = (u64)__float2uint_rz(fminf(qf, 1048576.0f));
        u64 p = q * d;
        q = (__umul64hi(q, d) != 0 || p > n) ? q - 1 : (n - p >= d ? q + 1 : q);
        p = q * d;
        q = (__umul64hi(q, d) != 0 || p > n) ? q - 1 : (n - p >= d ? q + 1 : q);
        const u64 q_all = (untouched >> r) & 1;
        const bool unconstrained = !on || (!all && (n == HQS_AMOUNT_MAX || fits_cap));
        big |= on && !all && !unconstrained && qf >= 1048576.0f;
        const u64 qr = all ? q_all : q;
        cnt = unconstrained ? cnt : (cnt < qr ? cnt : qr);
    }
    if (big) {                                  // rare: exact 64-bit divisions
        cnt = cap;
#pragma unroll
        for (int r = 0; r < RT; ++r) {
            if (!((used >> r) & 1)) continue;
            u64 q;
            if ((allm >> r) & 1) q = (untouched >> r) & 1;
            else if (fr[r] != HQS_AMOUNT_MAX) q = fr[r] / dv.amount[r];
            else continue;
            cnt = cnt < q ? cnt : q;
        }
    }
    return cnt;
}

// Narrow amounts (< 2^31): exact division by the invariant amount with a precomputed magic number (Granlund &
// Montgomery, "Division by Invariant Integers using Multiplication", fig. 4.1): for 1 <= d < 2^32, l = ceil(log2 d),
// m = floor(2^32 (2^l - d) / d) + 1, sh1 = min(l, 1), sh2 = max(l - 1, 0):  n / d = (t + ((n - t) >> sh1)) >> sh2 with
// t = umulhi(m, n), for every 0 <= n < 2^32.  A handful of integer instructions per resource, no fix-up, no slow path.
template <int RT>
__device__ __forceinline__ u64 fit_count(const u32 (&fr)[RT], u32 untouched, const VarT<RT, u32>& dv, u64 cap64) {
    u32 cnt = (u32)cap64;
    const u32 used = dv.used_mask, allm = dv.all_mask;
    // straight-line: the RT quotient chains are independent (ILP on the solver's critical path); an unused resource has
    // amount 0, magic 0, shifts 0 and is dropped by the final select
#pragma unroll
    for (int r = 0; r < RT; ++r) {
        const bool on = (used >> r) & 1, all = (allm >> r) & 1;
        const u32 n = fr[r];
        const u32 m = __float_as_uint(dv.rcpf[r]);
        const u32 s = (dv.shw[r >> 2] >> ((r & 3) * 8)) & 0xFFu;
        const u32 t = __umulhi(m, n);
        u32 q = (t + ((n - t) >> (s & 1u))) >> (s >> 1);
        q = n == 0xFFFFFFFFu ? 0xFFFFFFFFu : q;                      // unbounded free amount
        q = all ? ((untouched >> r) & 1u) : q;
        cnt = on ? (cnt < q ? cnt : q) : cnt;
    }
    return cnt;
}

template <int RT, typename AT>
__device__ __forceinline__ void take_from(AT (&fr)[RT], const VarT<RT, AT>& dv, u64 k) {
#pragma unroll
    for (int r = 0; r < RT; ++r) {
        if (!((dv.used_mask >> r) & 1)) continue;
        if ((dv.all_mask >> r) & 1) fr[r] = 0;                               // workerload.rs:162
        else if (fr[r] != AmountMax<AT>::value) fr[r] -= (AT)k * dv.amount[r];
    }
}

// ---- pack: one warp fills one worker (specification: tests/greedy_model.py::_pack_level step b) ----
// Runs on the worker CTAs of the tick kernel (blockIdx.x >= 1), on exact 64-bit amounts.
struct PackArgs {
    PackScratch pk;
    const u64* total_rw;     // [W][R]
    const u64* rem_time;     // [W]
    const uint8_t* blocked;  // [W][Q] or nullptr
    const uint8_t* excluded; // [W] or nullptr (workers taken out of the tick by the min-utilisation rule)
    const void* classes64;   // ClassT<RT, u64>[Q]
    u32 W, Q, R;
};

template <int RT>
__device__ void pack_body(const PackArgs& a, unsigned char* smem_dyn) {
    // per-warp scratch in the dynamic shared memory of the worker CTAs
    double* s_dom = reinterpret_cast<double*>(smem_dyn) + (size_t)(threadIdx.x >> 5) * PACK_MAX_CAND;
    const ClassT<RT>* classes = reinterpret_cast<const ClassT<RT>*>(a.classes64);
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const u32 n_pack_ctas = gridDim.x - 1;
    const u32 n_cand = __ldcg(a.pk.meta);
    // worker w is filled by CTA 1 + w % n_pack_ctas, warp w / n_pack_ctas: spreads the warps over the SMs
    for (u32 w = (blockIdx.x - 1) + warp * n_pack_ctas; w < a.W; w += n_pack_ctas * (blockDim.x >> 5)) {
        if (a.excluded && __ldcg(a.excluded + w)) {
#pragma unroll
            for (int j = 0; j < 2; ++j)
                if (lane + 32 * j < n_cand) a.pk.taken[(size_t)w * PACK_MAX_CAND + lane + 32 * j] = 0;
            continue;
        }
        u64 fr[RT], tot[RT];
#pragma unroll
        for (int r = 0; r < RT; ++r) {
            fr[r] = r < (int)a.R ? __ldcg(a.pk.fr + (size_t)w * a.R + r) : 0;
            tot[r] = r < (int)a.R ? a.total_rw[(size_t)w * a.R + r] : 0;
        }
        const u64 rem_time = a.rem_time[w];
        // exact u64 -> double through the 32-bit halves (one rounding, same value as a direct conversion)
        auto to_double = [](u64 x) -> double {
            return __dadd_rn(__dmul_rn(__uint2double_rn((u32)(x >> 32)), 4294967296.0), __uint2double_rn((u32)x));
        };
        // reciprocals once per worker / candidate: the per-iteration score is multiply-add only
        double inv_tot[RT];
#pragma unroll
        for (int r = 0; r < RT; ++r)
            inv_tot[r] = (tot[r] != 0 && tot[r] != HQS_AMOUNT_MAX) ? __ddiv_rn(1.0, to_double(tot[r])) : 0.0;
        // my two candidates
        u32 cls[2], var[2], gi[2], quota[2], taken[2], gs[2], ge[2];
        bool live[2];
        double inv_norm[2], dvec[2][RT];
        const VarT<RT>* dv[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const u32 ci = lane + 32 * j;
            live[j] = ci < n_cand;
            taken[j] = 0; quota[j] = 0; inv_norm[j] = 0.0; cls[j] = var[j] = gi[j] = 0; dv[j] = &classes[0].v[0];
            gs[j] = ge[j] = 0;
#pragma unroll
            for (int r = 0; r < RT; ++r) dvec[j][r] = 0.0;
            if (live[j]) {
                const u32 cd = __ldcg(a.pk.cand + ci);
                cls[j] = cd & 0xFFFFu; var[j] = (cd >> 16) & 0xFFu; gi[j] = cd >> 24;
                dv[j] = &classes[cls[j]].v[var[j]];
                gs[j] = ci - var[j];                                  // the variants of a group are consecutive candidates
                ge[j] = gs[j] + classes[cls[j]].n_variants;
                quota[j] = __ldcg(a.pk.quota + (size_t)w * PACK_MAX_CAND + gi[j]);
                const uint8_t blk = a.blocked ? a.blocked[(size_t)w * a.Q + cls[j]] : 0;
                live[j] = admissible(*dv[j], var[j], blk, rem_time);
                double s2 = 0.0;
#pragma unroll
                for (int r = 0; r < RT; ++r) {
                    if ((dv[j]->used_mask >> r) & 1) dvec[j][r] = __dmul_rn(to_double(dv[j]->amount[r]), inv_tot[r]);
                    s2 = __dadd_rn(s2, __dmul_rn(dvec[j][r], dvec[j][r]));
                }
                const double nrm = __dsqrt_rn(s2);
                inv_norm[j] = nrm > 0.0 ? __ddiv_rn(1.0, nrm) : 0.0;
            }
        }
        for (u32 it = 0; it < PACK_MAX_ITER; ++it) {
            double u[RT], inv_u[RT];
#pragma unroll
            for (int r = 0; r < RT; ++r) {
                u[r] = __dmul_rn(to_double(fr[r]), inv_tot[r]);
                inv_u[r] = __ddiv_rn(1.0, u[r]);                      // +inf where nothing is left
            }
            // a. per candidate: feasible? its dominant share of what the worker has left
            bool elig[2];
            double dom[2];
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                elig[j] = live[j] && quota[j] != 0;
                dom[j] = 0.0;
                if (elig[j]) {
#pragma unroll
                    for (int r = 0; r < RT; ++r) {
                        if (((dv[j]->used_mask >> r) & 1) && fr[r] != HQS_AMOUNT_MAX && dv[j]->amount[r] > fr[r]) elig[j] = false;
                        if (dvec[j][r] > 0.0) {
                            const double x = __dmul_rn(dvec[j][r], inv_u[r]);
                            dom[j] = x > dom[j] ? x : dom[j];
                        }
                    }
                }
                if (lane + 32 * j < PACK_MAX_CAND) s_dom[lane + 32 * j] = elig[j] ? dom[j] : -1.0;   // -1: not eligible
            }
            __syncwarp();
            // b. per group the eligible variant with the smallest share (ties: lower index) stays in the race
            double best_s = 0.0;
            u32 best_ci = ~0u;
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                if (!elig[j]) continue;
                const u32 ci = lane + 32 * j;
                bool win = true;
                for (u32 k = gs[j]; k < ge[j]; ++k) {
                    const double o = s_dom[k];
                    if (k != ci && o >= 0.0 && (o < dom[j] || (o == dom[j] && k < ci))) win = false;
                }
                if (!win) continue;
                double dot = 0.0;
#pragma unroll
                for (int r = 0; r < RT; ++r) dot = __dadd_rn(dot, __dmul_rn(dvec[j][r], u[r]));
                const double sc = __dmul_rn(dot, inv_norm[j]);
                if (best_ci == ~0u || sc > best_s) { best_s = sc; best_ci = ci; }   // j = 0 first: lower index wins ties
            }
            __syncwarp();
            // c. warp argmax: larger score, ties to the lower candidate index
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) {
                const double os = __shfl_xor_sync(0xffffffffu, best_s, d);
                const u32 oc = __shfl_xor_sync(0xffffffffu, best_ci, d);
                if (oc != ~0u && (best_ci == ~0u || os > best_s || (os == best_s && oc < best_ci))) { best_s = os; best_ci = oc; }
            }
            if (best_ci == ~0u) break;
            const u32 owner = best_ci & 31, oj = best_ci >> 5;
            u32 k = 0, ggi = 0;
            const VarT<RT>* mydv = oj ? dv[1] : dv[0];
            if (lane == owner) {
                const u32 q = oj ? quota[1] : quota[0];
                const u64 f = fit_count<RT>(fr, 0u, *mydv, q);        // levels with an `All` request are never packed
                const u32 chunk = q / PACK_CHUNK_DIV > 1 ? q / PACK_CHUNK_DIV : 1;
                k = (u32)(f < chunk ? f : chunk);
                if (oj) taken[1] += k; else taken[0] += k;
                ggi = oj ? gi[1] : gi[0];
            }
            k = __shfl_sync(0xffffffffu, k, owner);
            ggi = __shfl_sync(0xffffffffu, ggi, owner);
            // every lane applies the owner's amounts to its copy of the free vector
            const VarT<RT>* odv = (const VarT<RT>*)__shfl_sync(0xffffffffu, (unsigned long long)mydv, owner);
            take_from<RT, u64>(fr, *odv, k);
#pragma unroll
            for (int j = 0; j < 2; ++j)
                if (gi[j] == ggi && (lane + 32 * j) < n_cand) quota[j] = quota[j] >= k ? quota[j] - k : 0;
        }
#pragma unroll
        for (int j = 0; j < 2; ++j)
            if (lane + 32 * j < n_cand) a.pk.taken[(size_t)w * PACK_MAX_CAND + lane + 32 * j] = taken[j];
        if (lane == 0) {
#pragma unroll
            for (int r = 0; r < RT; ++r)
                if (r < (int)a.R) a.pk.fr[(size_t)w * a.R + r] = fr[r];
        }
    }
}
#endif  // __CUDACC__
