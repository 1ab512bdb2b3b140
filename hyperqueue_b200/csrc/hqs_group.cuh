// hqs_group.cuh — per-worker grouping of a tick's records on the device (hqs_tick_fetch_grouped).  Included by hqsched.cu.
//
// A stable counting sort of the flat record stream d_out[0..n) by
//     key = kind == 2 ? 2W : 2 * worker + (kind == 0)                                  (K = 2W + 1 keys)
// so that worker w's prefill records (kind 1) are out[off[2w] .. off[2w+1]), its assignments (kind 0) are
// out[off[2w+1] .. off[2w+2]), both in emission order, and the redirect records (kind 2) stay in a flat tail in emission order.
// Three plain launches on the context stream, run at fetch time when n is known on the host:
//   group_count_k    one CTA per tile of GROUP_TILE records: shared-memory histogram over the keys, one column of hist[key][tile]
//   group_scan_k     one warp per key: exclusive prefix over the tiles, in place; the block that finishes last (a ticket, nobody
//                    waits) scans the key totals into the offset table off[0 .. K]
//   group_scatter_k  stable rank of every record inside its tile without an atomic deciding an order: a warp owns 256
//                    consecutive records, the records of one key inside a warp step are ranked by lane (__match_any_sync), the
//                    steps by a per-warp counter in shared memory, the warps by a prefix over the 16 counters of the key
// The output is a function of the input alone: bit-identical from run to run.  Every loop is bounded by n, K or the tile count.

constexpr u32 GROUP_THREADS = 512;
constexpr u32 GROUP_WARPS = GROUP_THREADS / 32;
constexpr u32 GROUP_PER_THREAD = 8;
constexpr u32 GROUP_TILE = GROUP_THREADS * GROUP_PER_THREAD;          // records per CTA
constexpr u32 GROUP_WARP_SPAN = 32 * GROUP_PER_THREAD;               // consecutive records a scatter warp owns
constexpr u32 GROUP_SCAN_THREADS = 256;

// a record as the two words it is loaded as: x = task, y = worker | variant << 16 | kind << 24
__device__ __forceinline__ u32 group_key(u32 y, u32 W) {
    const u32 kind = y >> 24, worker = y & 0xFFFFu;
    return kind == 2 ? 2 * W : min(2 * worker + (kind == 0 ? 1u : 0u), 2 * W);
}

// adds the warp's records to the shared histogram: one add per distinct key of the step
__device__ __forceinline__ void group_hist_add(u32* hist, u32 key, bool valid, u32 lane) {
    const u32 peers = __match_any_sync(0xFFFFFFFFu, valid ? key : 0xFFFFFFFFu);
    if (valid && lane == (u32)__ffs(peers) - 1) atomicAdd(&hist[key], (u32)__popc(peers));
}

__global__ void __launch_bounds__(GROUP_THREADS) group_count_k(const hqs_assignment* __restrict__ in, u32 n, u32 W, u32 T,
                                                               u32* __restrict__ hist) {
    extern __shared__ u32 g_hist[];
    const u32 K = 2 * W + 1, tile = blockIdx.x, lane = threadIdx.x & 31;
    for (u32 k = threadIdx.x; k < K; k += GROUP_THREADS) g_hist[k] = 0;
    __syncthreads();
    // 16-byte loads, two records each (GROUP_TILE is even and the buffer is 256-byte aligned)
    const uint4* in2 = reinterpret_cast<const uint4*>(in);
    const u32 pair0 = tile * (GROUP_TILE / 2);
#pragma unroll
    for (u32 j = 0; j < GROUP_PER_THREAD / 2; ++j) {
        const u32 p = pair0 + j * GROUP_THREADS + threadIdx.x;
        const bool v0 = 2 * (u64)p < n, v1 = 2 * (u64)p + 1 < n;
        uint4 r = make_uint4(0, 0, 0, 0);
        if (v1) r = in2[p];
        else if (v0) r.y = reinterpret_cast<const uint2*>(in)[2 * (size_t)p].y;
        group_hist_add(g_hist, group_key(r.y, W), v0, lane);
        group_hist_add(g_hist, group_key(r.w, W), v1, lane);
    }
    __syncthreads();
    for (u32 k = threadIdx.x; k < K; k += GROUP_THREADS) hist[(size_t)k * T + tile] = g_hist[k];
}

__device__ __forceinline__ u32 warp_inclusive_scan(u32 v, u32 lane) {
#pragma unroll
    for (u32 d = 1; d < 32; d <<= 1) {
        const u32 o = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if (lane >= d) v += o;
    }
    return v;
}

__global__ void __launch_bounds__(GROUP_SCAN_THREADS) group_scan_k(u32* __restrict__ hist, u32 K, u32 T, u32* key_total,
                                                                   u32* __restrict__ off, u32* ticket) {
    __shared__ u32 s_warp[GROUP_SCAN_THREADS / 32];
    __shared__ u32 s_last;
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const u32 k = blockIdx.x * (GROUP_SCAN_THREADS / 32) + warp;
    if (k < K) {
        u32* row = hist + (size_t)k * T;
        u32 run = 0;
        for (u32 t0 = 0; t0 < T; t0 += 32) {
            const u32 t = t0 + lane;
            const u32 v = t < T ? row[t] : 0;
            const u32 incl = warp_inclusive_scan(v, lane);
            if (t < T) row[t] = run + incl - v;
            run += __shfl_sync(0xFFFFFFFFu, incl, 31);
        }
        if (lane == 0) key_total[k] = run;
    }
    // the block whose ticket is the last one has every key total before it: it alone goes on (no block waits for another)
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1u) == gridDim.x - 1 ? 1u : 0u;
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    u32 run = 0;
    for (u32 k0 = 0; k0 < K; k0 += GROUP_SCAN_THREADS) {
        const u32 kk = k0 + threadIdx.x;
        const u32 v = kk < K ? __ldcg(&key_total[kk]) : 0;
        const u32 incl = warp_inclusive_scan(v, lane);
        if (lane == 31) s_warp[warp] = incl;
        __syncthreads();
        u32 before = 0, all = 0;
        for (u32 w = 0; w < GROUP_SCAN_THREADS / 32; ++w) {
            before += w < warp ? s_warp[w] : 0;
            all += s_warp[w];
        }
        if (kk < K) off[kk] = run + before + incl - v;
        run += all;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        off[K] = run;
        *ticket = 0;                  // for the next fetch
    }
}

// dynamic shared memory of group_scatter_k: the tile's first output slot per key + the per-warp counters
inline size_t group_scatter_smem(u32 W) { return (size_t)(2 * W + 1) * (4 + GROUP_WARPS * 2); }

__global__ void __launch_bounds__(GROUP_THREADS) group_scatter_k(const hqs_assignment* __restrict__ in, u32 n, u32 W, u32 T,
                                                                 const u32* __restrict__ hist_excl, const u32* __restrict__ off,
                                                                 hqs_assignment* __restrict__ out) {
    extern __shared__ u32 g_smem[];
    const u32 K = 2 * W + 1, tile = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32* base = g_smem;                                                   // [K] first slot of the tile's records of the key
    unsigned short* cnt = reinterpret_cast<unsigned short*>(g_smem + K);  // [GROUP_WARPS][K], <= GROUP_TILE
    for (u32 k = threadIdx.x; k < K; k += GROUP_THREADS) base[k] = off[k] + hist_excl[(size_t)k * T + tile];
    for (u32 i = threadIdx.x; i < GROUP_WARPS * K; i += GROUP_THREADS) cnt[i] = 0;
    __syncthreads();
    unsigned short* mine = cnt + (size_t)warp * K;
    const u32 first = tile * GROUP_TILE + warp * GROUP_WARP_SPAN;
    const uint2* in1 = reinterpret_cast<const uint2*>(in);
    uint2 rec[GROUP_PER_THREAD];
    u32 key[GROUP_PER_THREAD], rank[GROUP_PER_THREAD];
    // rank inside the warp's span: the records of earlier steps (the counter), then the lower lanes of this step
#pragma unroll
    for (u32 j = 0; j < GROUP_PER_THREAD; ++j) {
        const u32 i = first + j * 32 + lane;
        const bool valid = i < n;
        rec[j] = valid ? in1[i] : make_uint2(0, 0);
        key[j] = valid ? group_key(rec[j].y, W) : 0xFFFFFFFFu;
        const u32 peers = __match_any_sync(0xFFFFFFFFu, key[j]);
        const u32 prior = valid ? mine[key[j]] : 0;
        __syncwarp();
        if (valid && lane == (u32)__ffs(peers) - 1) mine[key[j]] = (unsigned short)(prior + __popc(peers));
        __syncwarp();
        rank[j] = prior + __popc(peers & ((1u << lane) - 1));
    }
    __syncthreads();
    // counters -> exclusive prefix over the warps of the tile, key by key
    for (u32 k = threadIdx.x; k < K; k += GROUP_THREADS) {
        u32 run = 0;
#pragma unroll
        for (u32 w = 0; w < GROUP_WARPS; ++w) {
            const u32 c = cnt[(size_t)w * K + k];
            cnt[(size_t)w * K + k] = (unsigned short)run;
            run += c;
        }
    }
    __syncthreads();
    uint2* out1 = reinterpret_cast<uint2*>(out);
#pragma unroll
    for (u32 j = 0; j < GROUP_PER_THREAD; ++j)
        if (key[j] != 0xFFFFFFFFu) out1[base[key[j]] + mine[key[j]] + rank[j]] = rec[j];
}
