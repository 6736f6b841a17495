// 3dgrut_b200/csrc/gut_binning.cu -- G2 / G4 / G5 of the 3DGUT forward without a global sort (ours; no library calls).
//
// Reference (threedgut_tracer/src/gutRenderer.cu:303-373): inclusive scan of the per-particle tile counts (CUB), host read of the
// total, expand into 64-bit (tile << 32 | depth) keys, ONE stable 44-bit CUB radix sort of all I keys, tile ranges from the sorted
// stream.  The order it defines inside a tile is (depth bits, particle index) -- a stable sort of keys emitted in particle order.
//
// Here (DESIGN.md section 6):
//   project        counts every particle's tiles AND bumps a per-tile histogram           (gut_project.cu, atomics on T counters)
//   tile_scan      reduce-then-scan of the histogram across the GPU -> tile ranges (= G5, no pass over the keys), hit-word slices,
//                  heaviest-first tile order, total I and the capacity check on the device
//   expand_place   every (particle, tile) pair is dropped into its tile's slice at an atomically claimed slot as the 64-bit key
//                  (depth bits << 32 | particle index)                                      (gut_project.cu)
//   tile_sort      one CTA per tile sorts its slice by that key: a stable LSD radix sort over the depth bits (8 bits a pass, passes
//                  with a single digit skipped; a slice of up to 4096 keys is sorted in shared memory, a longer one ping-pongs
//                  through the L2) + a fix-up of equal-depth runs by particle index
//                  (a first version used a bitonic network: 125 M compare-exchanges at C2 cost 0.13 ms, 2.0 ms at C3 -- replaced)
// The keys are unique inside a tile (a particle enters a tile once), so the result is exactly the reference's order whatever order
// the atomics claimed the slots in; only sorted artefacts are observable and they stay bit-identical (tests/test_gut_parity_gpu.py).
// Work: I x 8 B written once, sorted in place on chip; no N-sized depth sort, no scan over N, no multi-pass radix sort over I.
#include <cstdlib>

#include "gut_common.cuh"

namespace gutb200 {

namespace {

constexpr unsigned kFullMask = 0xFFFFFFFFu;

// ----------------------------------------------------------------------------------------------------------
// tile_scan: a reduce-then-scan across the GPU, one tile per thread.  Every tile owns kTileSubs sub-counters (a particle bumps
// sub-counter `particle & (kTileSubs - 1)`): the atomics of a hot tile -- thousands of increments of one address serialise in the L2 --
// spread over kTileSubs addresses, and the slots of a tile's slice are claimed per sub-bucket the same way.  counts[T][kTileSubs] ->
// ranges[T][2] ((0, 0) for an empty tile, as the reference's zero-filled range buffer reads), sub_base[T][kTileSubs] (first slot of each
// sub-bucket), chunk_base[T], order[T] (decreasing list length, bucketed by log2), fill[T][kTileSubs] = 0, totals[0] = I, totals[1] = 1 if
// I exceeds the capacity of the key buffers (empty ranges are published then and the host re-launches the dependent kernels after
// growing the buffers).
//   tile_scan_reduce  CTA b: the list total, the hit-word chunk total and the 34 length-bucket counts of its kScanTiles tiles -> parts[b]
//   tile_scan_write   CTA b: its offsets from parts[0, b) and the grid totals from all parts, then every per-tile output
// (A single CTA of 1024 threads did both passes before: 0.036 ms at C2 on an H100, bound by the latency of its dependent passes with 131
// SMs idle.)  The order of the tiles inside one length bucket depends on the shared-memory atomics that hand out the slots; nothing
// observable depends on it -- `order` only schedules the tiles of the sort and render grids.

constexpr int kScanTiles = 256;                 // tiles (= threads) per CTA
constexpr int kScanBuckets = 34;                // length buckets: clz(count) + 1 in 1..33 (33 = empty tile); index 0 unused
constexpr int kScanPart = 2 + kScanBuckets;     // words per CTA in `parts`: list total, chunk total, bucket counts

// the tile's list length from its 16 sub-counters (four 16-byte loads); its bucket (__clz(0) = 32 -> last bucket, long lists first)
__device__ __forceinline__ uint32_t tile_count(const uint32_t* __restrict__ counts, int t, uint4 v[4]) {
    const uint4* c4 = reinterpret_cast<const uint4*>(counts + static_cast<size_t>(t) * kTileSubs);
    v[0] = c4[0]; v[1] = c4[1]; v[2] = c4[2]; v[3] = c4[3];
    return (v[0].x + v[0].y + v[0].z + v[0].w) + (v[1].x + v[1].y + v[1].z + v[1].w) + (v[2].x + v[2].y + v[2].z + v[2].w) +
           (v[3].x + v[3].y + v[3].z + v[3].w);
}

// exclusive block scan of (a, b) over the CTA's threads in thread order
__device__ __forceinline__ void scan_pair(uint32_t a, uint32_t b, uint32_t& ex_a, uint32_t& ex_b, uint32_t& tot_a, uint32_t& tot_b) {
    __shared__ uint32_t w_a[kScanTiles / 32], w_b[kScanTiles / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t ia = a, ib = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t x = __shfl_up_sync(kFullMask, ia, o), y = __shfl_up_sync(kFullMask, ib, o);
        if (lane >= o) {
            ia += x;
            ib += y;
        }
    }
    if (lane == 31) {
        w_a[warp] = ia;
        w_b[warp] = ib;
    }
    __syncthreads();
    uint32_t ra = 0, rb = 0;
    tot_a = 0;
    tot_b = 0;
#pragma unroll
    for (int w = 0; w < kScanTiles / 32; ++w) {
        if (w == warp) {
            ra = tot_a;
            rb = tot_b;
        }
        tot_a += w_a[w];
        tot_b += w_b[w];
    }
    ex_a = ra + ia - a;
    ex_b = rb + ib - b;
}

__global__ void __launch_bounds__(kScanTiles) tile_scan_reduce_kernel(int num_tiles, const uint32_t* __restrict__ counts,
                                                                      uint32_t* __restrict__ parts) {
    static_assert(kTileSubs == 16, "a tile's sub-counters are four 16-byte loads");
    __shared__ uint32_t hist[kScanBuckets];
    if (threadIdx.x < kScanBuckets) hist[threadIdx.x] = 0;
    __syncthreads();
    const int t = blockIdx.x * kScanTiles + threadIdx.x, lane = threadIdx.x & 31;
    const bool live = t < num_tiles;
    uint4 v[4];
    const uint32_t c = live ? tile_count(counts, t, v) : 0u;
    // The length buckets are few and most tiles fall into two or three of them, so a warp's lanes that land in the same bucket go through
    // ONE shared-memory atomic (match.any + population count) instead of serialising on its address
    const int bucket = live ? __clz(c) + 1 : 64 + lane;
    const unsigned peers = __match_any_sync(kFullMask, bucket);
    if (live && (peers & ((1u << lane) - 1u)) == 0u) atomicAdd(&hist[bucket], static_cast<uint32_t>(__popc(peers)));
    uint32_t ex_n, ex_c, tot_n, tot_c;
    scan_pair(c, (c + 31u) >> 5, ex_n, ex_c, tot_n, tot_c);   // ends after a barrier: hist is complete
    uint32_t* p = parts + static_cast<size_t>(blockIdx.x) * kScanPart;
    if (threadIdx.x == 0) {
        p[0] = tot_n;
        p[1] = tot_c;
    }
    if (threadIdx.x < kScanBuckets) p[2 + threadIdx.x] = hist[threadIdx.x];
}

__global__ void __launch_bounds__(kScanTiles) tile_scan_write_kernel(int num_tiles, const uint32_t* __restrict__ counts, uint32_t capacity,
                                                                     const uint32_t* __restrict__ parts, uint32_t* __restrict__ ranges,
                                                                     uint32_t* __restrict__ sub_base, uint32_t* __restrict__ chunk_base,
                                                                     uint32_t* __restrict__ order, uint32_t* __restrict__ fill,
                                                                     uint32_t* __restrict__ totals) {
    __shared__ uint32_t s_before[kScanPart], s_all[kScanPart];   // sums over the CTAs before this one / over all CTAs
    __shared__ uint32_t hist[kScanBuckets];                     // -> next free slot of each bucket in `order` for this CTA's tiles
    const int t = blockIdx.x * kScanTiles + threadIdx.x, lane = threadIdx.x & 31;
    if (threadIdx.x < kScanPart) {
        uint32_t before = 0, all = 0;
        for (int b = 0; b < static_cast<int>(gridDim.x); ++b) {
            const uint32_t x = parts[static_cast<size_t>(b) * kScanPart + threadIdx.x];
            before += b < static_cast<int>(blockIdx.x) ? x : 0u;
            all += x;
        }
        s_before[threadIdx.x] = before;
        s_all[threadIdx.x] = all;
    }
    __syncthreads();
    if (threadIdx.x == 0) {   // bucket b's tiles start after every tile of buckets < b and after bucket b's tiles of the CTAs before
        uint32_t run = 0;
        for (int b = 1; b < kScanBuckets; ++b) {
            hist[b] = run + s_before[2 + b];
            run += s_all[2 + b];
        }
    }
    const uint32_t total = s_all[0];
    const bool overflow = total > capacity;   // the lists do not fit the key buffer: publish empty ranges, the host grows and re-queues
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        totals[0] = total;
        totals[1] = overflow ? 1u : 0u;
    }
    const bool live = t < num_tiles;
    uint4 v[4];
    const uint32_t c = live ? tile_count(counts, t, v) : 0u;
    uint32_t ex_n, ex_c, tot_n, tot_c;
    scan_pair(c, (c + 31u) >> 5, ex_n, ex_c, tot_n, tot_c);   // ends after a barrier: hist is set up
    if (live) {
        // the thread that owns a tile lays out its sub-buckets itself and writes them with 16-byte stores
        uint32_t r = s_before[0] + ex_n;
        const uint32_t first = r;
        uint4 b[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            b[q].x = r; r += v[q].x; b[q].y = r; r += v[q].y; b[q].z = r; r += v[q].z; b[q].w = r; r += v[q].w;
        }
        uint4* sb = reinterpret_cast<uint4*>(sub_base + static_cast<size_t>(t) * kTileSubs);
        sb[0] = b[0]; sb[1] = b[1]; sb[2] = b[2]; sb[3] = b[3];
        const uint32_t fill0 = overflow ? 0xC0000000u : 0u;   // a huge fill level makes every claim fall outside its sub-bucket
        const uint4 fill4 = make_uint4(fill0, fill0, fill0, fill0);
        uint4* fl = reinterpret_cast<uint4*>(fill + static_cast<size_t>(t) * kTileSubs);
        fl[0] = fill4; fl[1] = fill4; fl[2] = fill4; fl[3] = fill4;
        // empty tile (or nothing fits): (0, 0) like the reference's zero-filled range buffer
        reinterpret_cast<uint2*>(ranges)[t] = (overflow || c == 0u) ? make_uint2(0u, 0u) : make_uint2(first, r);
        chunk_base[t] = overflow ? 0u : s_before[1] + ex_c;
    }
    const int bucket = live ? __clz(c) + 1 : 64 + lane;
    const unsigned peers = __match_any_sync(kFullMask, bucket);
    const int leader = __ffs(peers) - 1;
    uint32_t slot = 0;
    if (live && lane == leader) slot = atomicAdd(&hist[bucket], static_cast<uint32_t>(__popc(peers)));
    slot = __shfl_sync(kFullMask, slot, leader);
    if (live) order[slot + __popc(peers & ((1u << lane) - 1u))] = static_cast<uint32_t>(t);
}

// ----------------------------------------------------------------------------------------------------------
// tile_sort: one CTA per tile sorts the tile's slice of 64-bit keys (depth bits << 32 | particle) -- a least-significant-digit radix
// sort over the 32 depth bits, 8 bits a pass, ping-ponging between the key buffer and its twin (both stay in the L2: a slice is a few
// tens of KB), shared memory holding only the digit counters.  Each of the CTA's warps owns a contiguous segment of the slice and
// keeps its elements in order (32 at a time: `match.any` groups equal digits, the group's first lane claims their slots), so a pass is
// stable; passes in which every key carries the same digit (typically the exponent byte) are skipped.  The depth order the passes
// produce is completed to (depth, particle) order by a fix-up of runs of EQUAL depth bits -- duplicates of a position, e.g. freshly
// cloned Gaussians; the slots were claimed in arbitrary order, so the sort cannot rely on stability for them.

//
// A slice of at most kStageKeys keys (every tile of C2) is sorted in shared memory instead: it is loaded once, each pass reads the warp's
// segment into registers, ranks it and scatters it back into the same shared buffer (the reads of a pass end at the barriers before its
// scatter, so one buffer suffices), the fix-up runs there, and the values are written once.  Longer slices (C3: 6-30 k keys) keep the
// L2 ping-pong.  The CTA picks its path from n, so the choice is uniform across it.

constexpr int kSortThreads = 512, kSortWarps = kSortThreads / 32;   // 16 warps per tile: the long lists (6-30 k keys at C3) are latency-bound
constexpr int kSortUnroll = 4;                                      // keys in flight per lane in the count / scatter loops
// Staged slices: 4096 keys = 32 KB of dynamic shared memory, 8 keys per lane in registers.  With the 16 KB of digit counters a CTA takes
// 48 KB, so the three CTAs the register count allows per SM still fit (the longest C2 list is about 3.6 k keys).
constexpr int kStageKeys = 4096, kStagePerLane = kStageKeys / kSortThreads;

// threads 0..255: digit d's total over the aw counter rows, an exclusive scan over the digits, then the first slot of (warp, d).
// Returns true (uniformly) when every key carries one digit: the pass would be the identity and is skipped.  Ends on a barrier.
__device__ __forceinline__ bool scan_digits(uint32_t (*s_cnt)[256], uint32_t* s_tot, int* s_flag, int aw, uint32_t n) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, d = threadIdx.x;
    uint32_t tot = 0, incl = 0;
    if (d < 256) {
        for (int w = 0; w < aw; ++w) tot += s_cnt[w][d];
        if (tot == n) *s_flag = 1;
        incl = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(kFullMask, incl, o);
            if (lane >= o) incl += v;
        }
        if (lane == 31) s_tot[warp] = incl;   // totals of the 8 groups of 32 digits
    }
    __syncthreads();
    const bool skip = *s_flag != 0;   // uniform across the CTA
    if (!skip && d < 256) {
        uint32_t run = incl - tot;
        for (int w = 0; w < warp; ++w) run += s_tot[w];
        for (int w = 0; w < aw; ++w) {
            const uint32_t c = s_cnt[w][d];
            s_cnt[w][d] = run;
            run += c;
        }
    }
    __syncthreads();
    return skip;
}

// Slot of this lane's key among the warp's 32 (in lane order, so the pass is stable); `have` is warp-divergent, the call warp-uniform.
template <bool BALLOT>
__device__ __forceinline__ uint32_t rank_key(uint32_t* cnt_row, unsigned long long k, int shift, bool have) {
    const int lane = threadIdx.x & 31;
    const uint32_t dg = have ? (static_cast<uint32_t>(k >> shift) & 255u) : 256u + lane;  // idle lanes: unique pseudo-digits
    unsigned peers;
    if (BALLOT) {  // lanes with the same 8-bit digit, from one ballot per bit (the multi-split CUB's ranking uses)
        peers = __ballot_sync(kFullMask, have);
#pragma unroll
        for (int b = 0; b < 8; ++b) {
            const bool bit = (dg >> b) & 1u;
            const unsigned bal = __ballot_sync(kFullMask, bit);
            peers &= bit ? bal : ~bal;
        }
        if (!have) peers = 1u << lane;
    } else {
        peers = __match_any_sync(kFullMask, dg);
    }
    const int leader = __ffs(peers) - 1;
    uint32_t slot = 0;
    if (have && lane == leader) slot = atomicAdd(&cnt_row[dg], static_cast<uint32_t>(__popc(peers)));
    slot = __shfl_sync(kFullMask, slot, leader);
    return slot + __popc(peers & ((1u << lane) - 1u));
}

// `a[0, n)` is in depth order.  Runs of EQUAL depth bits are ordered by particle index by the thread whose element starts the run (runs
// are disjoint, a run is two or three keys long; a serial walk by one thread cost milliseconds here: every second C3 tile has such a pair)
__device__ __forceinline__ void fix_equal_depth_runs(unsigned long long* a, uint32_t n) {
    for (uint32_t i = threadIdx.x; i + 1 < n; i += kSortThreads) {
        const unsigned long long x = a[i];
        if ((x >> 32) != (a[i + 1] >> 32)) continue;
        if (i > 0 && (a[i - 1] >> 32) == (x >> 32)) continue;  // inside a run: its first element's thread handles it
        uint32_t e = i + 2;
        while (e < n && (a[e] >> 32) == (x >> 32)) ++e;
        for (uint32_t p = i + 1; p < e; ++p) {  // insertion sort of a[i .. e)
            const unsigned long long k = a[p];
            uint32_t q = p;
            while (q > i && a[q - 1] > k) {
                a[q] = a[q - 1];
                --q;
            }
            a[q] = k;
        }
    }
}

template <bool BALLOT>
__global__ void __launch_bounds__(kSortThreads) tile_sort_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ ranges,
                                                                 const uint32_t* __restrict__ totals, unsigned long long* keys,
                                                                 unsigned long long* keys_alt, uint32_t* __restrict__ sorted_values) {
    __shared__ uint32_t s_cnt[kSortWarps][256];   // per-warp digit counts -> running slot of (warp, digit)
    __shared__ uint32_t s_tot[8];
    __shared__ int s_flag;
    extern __shared__ unsigned long long s_keys[];  // kStageKeys entries: the staged slice
    if (totals[1] != 0u) return;  // capacity exceeded: the host grows the buffers and launches again
    const uint32_t tile = order[blockIdx.x];
    const uint32_t begin = ranges[tile * 2], n = ranges[tile * 2 + 1] - begin;
    if (n == 0u) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long* src = keys + begin;
    unsigned long long* dst = keys_alt + begin;
    // Short lists use fewer warps (>= 128 keys each): the per-pass fixed cost -- zeroing, summing and scanning one counter row per warp --
    // scales with the warps that take part, and most C2 tiles hold a few hundred keys.
    const int aw = static_cast<int>(min(static_cast<uint32_t>(kSortWarps), max(1u, (n + 127u) / 128u)));
    // warp w < aw owns elements [w * seg, min(n, (w + 1) * seg)), seg a multiple of 32 (at most 32 * kStagePerLane when n <= kStageKeys)
    const uint32_t seg = ((n + aw - 1) / aw + 31u) & ~31u;
    const uint32_t w0 = min(n, warp * seg), w1 = min(n, w0 + seg);

    if (n <= static_cast<uint32_t>(kStageKeys)) {
        for (uint32_t i = threadIdx.x; i < n; i += kSortThreads) s_keys[i] = src[i];
        for (int shift = 32; shift < 64; shift += 8) {
            for (int i = threadIdx.x; i < aw * 256; i += kSortThreads) (&s_cnt[0][0])[i] = 0u;
            if (threadIdx.x == 0) s_flag = 0;
            __syncthreads();   // also: the previous pass's scatter (or the load) is complete
            unsigned long long k[kStagePerLane];
#pragma unroll
            for (int u = 0; u < kStagePerLane; ++u) {
                const uint32_t i = w0 + u * 32 + lane;
                k[u] = i < w1 ? s_keys[i] : 0ull;
                if (i < w1) atomicAdd(&s_cnt[warp][static_cast<uint32_t>(k[u] >> shift) & 255u], 1u);
            }
            __syncthreads();
            if (scan_digits(s_cnt, s_tot, &s_flag, aw, n)) continue;
#pragma unroll
            for (int u = 0; u < kStagePerLane; ++u) {   // 32 keys at a time, in order: the pass is stable
                if (w0 + u * 32 >= w1) break;           // warp-uniform
                const bool have = w0 + u * 32 + lane < w1;
                const uint32_t slot = rank_key<BALLOT>(s_cnt[warp], k[u], shift, have);
                if (have) s_keys[slot] = k[u];
            }
            __syncthreads();   // the counters are zeroed next: every warp is done claiming slots
        }
        fix_equal_depth_runs(s_keys, n);
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < n; i += kSortThreads) sorted_values[begin + i] = static_cast<uint32_t>(s_keys[i]);
        return;
    }

    for (int shift = 32; shift < 64; shift += 8) {
        for (int i = threadIdx.x; i < aw * 256; i += kSortThreads) (&s_cnt[0][0])[i] = 0u;
        if (threadIdx.x == 0) s_flag = 0;
        __syncthreads();
        for (uint32_t i0 = w0; i0 < w1; i0 += 32 * kSortUnroll) {  // digit counts of this warp's segment, kSortUnroll loads in flight
            unsigned long long k[kSortUnroll];
#pragma unroll
            for (int u = 0; u < kSortUnroll; ++u) {
                const uint32_t i = i0 + u * 32 + lane;
                k[u] = i < w1 ? src[i] : ~0ull;
            }
#pragma unroll
            for (int u = 0; u < kSortUnroll; ++u)
                if (i0 + u * 32 + lane < w1) atomicAdd(&s_cnt[warp][static_cast<uint32_t>(k[u] >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (scan_digits(s_cnt, s_tot, &s_flag, aw, n)) continue;
        for (uint32_t i0 = w0; i0 < w1; i0 += 32 * kSortUnroll) {
            unsigned long long k[kSortUnroll];
#pragma unroll
            for (int u = 0; u < kSortUnroll; ++u) {
                const uint32_t i = i0 + u * 32 + lane;
                k[u] = i < w1 ? src[i] : 0ull;
            }
#pragma unroll
            for (int u = 0; u < kSortUnroll; ++u) {   // 32 keys at a time, in order: the pass is stable
                if (i0 + u * 32 >= w1) break;         // warp-uniform
                const bool have = i0 + u * 32 + lane < w1;
                const uint32_t slot = rank_key<BALLOT>(s_cnt[warp], k[u], shift, have);
                if (have) dst[slot] = k[u];
            }
        }
        __syncthreads();
        unsigned long long* t = src;
        src = dst;
        dst = t;
    }
    // `src` holds the slice in depth order
    fix_equal_depth_runs(src, n);
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < n; i += kSortThreads) sorted_values[begin + i] = static_cast<uint32_t>(src[i]);
}

// test-only: the reference's sorted 64-bit keys (tile << 32 | depth bits), rebuilt per tile from the sorted values
__global__ void __launch_bounds__(256) synth_tile_keys_kernel(const uint32_t* __restrict__ ranges, const uint32_t* __restrict__ vals,
                                                              const float* __restrict__ depth, uint64_t* __restrict__ out) {
    const uint32_t tile = blockIdx.x;
    const uint32_t begin = ranges[tile * 2], end = ranges[tile * 2 + 1];
    for (uint32_t k = begin + threadIdx.x; k < end; k += blockDim.x)
        out[k] = (static_cast<uint64_t>(tile) << 32) | __float_as_uint(depth[vals[k]]);
}

}  // namespace

size_t tile_scan_parts_words(int num_tiles) { return static_cast<size_t>(max(1, (num_tiles + kScanTiles - 1) / kScanTiles)) * kScanPart; }

void launch_tile_scan(cudaStream_t s, int num_tiles, const uint32_t* counts, uint32_t capacity, uint32_t* ranges, uint32_t* sub_base,
                      uint32_t* chunk_base, uint32_t* order, uint32_t* fill, uint32_t* totals, uint32_t* parts) {
    const int blocks = max(1, (num_tiles + kScanTiles - 1) / kScanTiles);
    tile_scan_reduce_kernel<<<blocks, kScanTiles, 0, s>>>(num_tiles, counts, parts);
    tile_scan_write_kernel<<<blocks, kScanTiles, 0, s>>>(num_tiles, counts, capacity, parts, ranges, sub_base, chunk_base, order, fill, totals);
}

// heaviest tiles come first in `order`: the long lists start before the bulk of the short ones
cudaError_t launch_tile_sort(cudaStream_t s, int num_tiles, const uint32_t* order, const uint32_t* ranges, const uint32_t* totals,
                             unsigned long long* keys, unsigned long long* keys_alt, uint32_t* sorted_values) {
    if (num_tiles <= 0) return cudaSuccess;
    static const bool use_match = [] { const char* e = std::getenv("GUTB200_SORT_MATCH"); return e && std::atoi(e) != 0; }();  // A/B switch
    constexpr size_t kStageBytes = kStageKeys * sizeof(unsigned long long);
    static const cudaError_t opt_in = [] {   // static + dynamic shared memory exceeds the default 48 KB per CTA
        cudaError_t e = cudaFuncSetAttribute(tile_sort_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kStageBytes));
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(tile_sort_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kStageBytes));
        return e;
    }();
    if (opt_in != cudaSuccess) return opt_in;
    if (use_match)
        tile_sort_kernel<false><<<num_tiles, kSortThreads, kStageBytes, s>>>(order, ranges, totals, keys, keys_alt, sorted_values);
    else
        tile_sort_kernel<true><<<num_tiles, kSortThreads, kStageBytes, s>>>(order, ranges, totals, keys, keys_alt, sorted_values);
    return cudaGetLastError();
}

void launch_synth_tile_keys(cudaStream_t s, int num_tiles, const uint32_t* ranges, const uint32_t* vals, const float* depth, uint64_t* out) {
    if (num_tiles <= 0) return;
    synth_tile_keys_kernel<<<num_tiles, 256, 0, s>>>(ranges, vals, depth, out);
}

}  // namespace gutb200
