// String interning (easyrag_b200/vocab.py): the id a Python dict filled in first-seen order gives each string, and the
// index of its first occurrence, for batches of UTF-8 strings joined by NUL.  DESIGN.md §4.9.
//
// Per chunk of n strings (global indices g0 .. g0 + n):
//   1. bounds:  a scan over the bytes turns the NUL separators into string starts.
//   2. probe:   every string is hashed (a thread per string of <= 32 bytes, a warp per longer one) and inserted into an
//               open-addressing table that persists across chunks.  A slot holds a representative (an id, or a string
//               of the current chunk), its hash and the smallest global index seen.  Equal hashes are only a filter:
//               a slot is matched by byte equality with its representative, so a collision never merges two strings.
//   3. order:   a string is new iff its slot's first index is its own index; a scan over those flags gives each new
//               string its rank, so id = vocabulary size + rank is first-seen order without a sort.
//   4. publish: new slots take their ids, new strings' bytes go to the arena (bytes of id i at
//               arena_off[i] .. arena_off[i + 1]), and every string reads its id through its slot.
// Lookup runs 1 and 2 without inserting and writes -1 for a string the table does not hold.
#include <algorithm>
#include <climits>
#include "ezr_common.cuh"
#include "../../include/easyrag_b200.h"

namespace ezr {

constexpr uint64_t kP61 = (1ull << 61) - 1;                 // polynomial hash modulus (a Mersenne prime)
constexpr uint64_t kHashBase = 0x0B5AD4ECEDA1CE2Bull & kP61;
constexpr unsigned long long kHashUnset = ~0ull;           // slot hash before its claimer stores it
constexpr long long kRepEmpty = -1;                        // slot representative: -1 empty, >= 0 an id,
                                                           // <= -2 string -2 - r of the current chunk
constexpr int kShortMax = 32;                              // longer strings are hashed and compared by a warp
constexpr int kHdr = 8;                                    // table header: [0] capacity, [1] hash bits
constexpr int kThreads = 256;
constexpr int kScanItems = 16;
constexpr int64_t kScanTile = (int64_t)kThreads * kScanItems;
constexpr int kTopThreads = 1024;
constexpr int64_t kMaxChunkBytes = (1ll << 32) - 1;        // the order scan packs byte offsets into 32 bits

static thread_local int g_vocab_bits = 64;                 // ezr_vocab_set_hash_bits: tables created afterwards

// ------------------------------------------------------------------------------------------------ hashing ----
__device__ __forceinline__ uint64_t mulmod61(uint64_t a, uint64_t b) {
    const uint64_t lo = a * b, hi = __umul64hi(a, b);        // a, b < 2^61: the product is < 2^122
    uint64_t r = (lo & kP61) + ((lo >> 61) | (hi << 3));
    r = (r & kP61) + (r >> 61);
    return r >= kP61 ? r - kP61 : r;
}
__device__ __forceinline__ uint64_t addmod61(uint64_t a, uint64_t b) {
    const uint64_t r = a + b;
    return r >= kP61 ? r - kP61 : r;
}
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
    x ^= x >> 27; x *= 0x94d049bb133111ebull;
    return x ^ (x >> 31);
}
// H(s) = sum (s[i] + 1) * B^(len-1-i) mod P, then mixed with the length and cut to the table's hash bits
__device__ __forceinline__ uint64_t finish_hash(uint64_t h, int64_t len, int bits) {
    const uint64_t x = mix64(h ^ ((uint64_t)len * 0x9E3779B97F4A7C15ull));
    return bits >= 64 ? x : (x & ((1ull << bits) - 1));
}
__device__ __forceinline__ uint64_t hash_thread(const uint8_t* p, int64_t len) {
    uint64_t h = 0;
    for (int64_t i = 0; i < len; ++i) h = addmod61(mulmod61(h, kHashBase), (uint64_t)p[i] + 1);
    return h;
}
// each lane hashes one contiguous segment (h, B^len); a shuffle tree joins them in lane order:
// H(x ++ y) = H(x) * B^|y| + H(y).  Every lane returns the whole string's H.
__device__ __forceinline__ uint64_t hash_warp(const uint8_t* p, int64_t len, int lane) {
    const int64_t seg = (len + 31) / 32, lo = min(len, lane * seg), hi = min(len, lo + seg);
    uint64_t h = 0, pw = 1;
    for (int64_t i = lo; i < hi; ++i) {
        h = addmod61(mulmod61(h, kHashBase), (uint64_t)p[i] + 1);
        pw = mulmod61(pw, kHashBase);
    }
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t h2 = __shfl_down_sync(0xffffffffu, h, d), p2 = __shfl_down_sync(0xffffffffu, pw, d);
        if ((lane & (2 * d - 1)) == 0 && lane + d < 32) {
            h = addmod61(mulmod61(h, p2), h2);
            pw = mulmod61(pw, p2);
        }
    }
    return __shfl_sync(0xffffffffu, h, 0);
}
template <bool kWarp>
__device__ __forceinline__ bool bytes_equal(const uint8_t* a, const uint8_t* b, int64_t len, int lane) {
    if (!kWarp) {
        for (int64_t i = 0; i < len; ++i)
            if (a[i] != b[i]) return false;
        return true;
    }
    bool diff = false;
    for (int64_t i = lane; i < len && !diff; i += 32) diff = a[i] != b[i];
    return !__any_sync(0xffffffffu, diff);
}

// ------------------------------------------------------------------------------------------------- table ----
struct Str {
    const uint8_t* p;
    int64_t len;
};

struct Table {
    long long* rep;               // [cap]
    unsigned long long* hash;     // [cap]
    long long* first;             // [cap] smallest global index of the slot's string
    int64_t mask;
    __host__ Table(void* base, int64_t cap) {
        long long* t = (long long*)base + kHdr;
        rep = t;
        hash = (unsigned long long*)(t + cap);
        first = t + 2 * cap;
        mask = cap - 1;
    }
};

struct Chunk {
    const uint8_t* bytes;
    const int64_t* starts;        // [n] byte offset of every string; string s ends at starts[s + 1] - 1 or n_bytes
    int64_t n, n_bytes;
    const uint8_t* arena;
    const int64_t* arena_off;
    __device__ __forceinline__ Str str(int64_t s) const {
        const int64_t a = starts[s], e = s + 1 < n ? starts[s + 1] - 1 : n_bytes;
        return {bytes + a, e - a};
    }
    __device__ __forceinline__ Str rep_str(long long r) const {
        if (r >= 0) {
            const int64_t a = arena_off[r];
            return {arena + a, arena_off[r + 1] - a};
        }
        return str(-2 - r);
    }
};

__device__ __forceinline__ int64_t slot_start(uint64_t h, int64_t mask) { return (int64_t)(mix64(h + 0x632BE59BD9B4E019ull) & (uint64_t)mask); }

// The slot holding string s (claimed for it when kInsert and no slot holds it), or -1 on a lookup miss.  A claim
// stores the representative first (the CAS) and the hash after it; a prober that sees the representative before the
// hash compares bytes, so the order of the two stores never decides a match.  The caller keeps the load factor at
// most 1/2, so an empty slot ends every probe.
template <bool kWarp, bool kInsert>
__device__ int64_t probe(const Table& t, const Chunk& c, Str s, uint64_t h, long long my_rep, int lane) {
    int64_t slot = slot_start(h, t.mask);
    while (true) {
        long long r = 0;
        unsigned long long hs = 0;
        int claimed = 0;
        if (!kWarp || lane == 0) {
            r = ((volatile long long*)t.rep)[slot];
            if (kInsert && r == kRepEmpty) {
                r = (long long)atomicCAS((unsigned long long*)&t.rep[slot], (unsigned long long)kRepEmpty,
                                         (unsigned long long)my_rep);
                if (r == kRepEmpty) {
                    claimed = 1;
                    ((volatile unsigned long long*)t.hash)[slot] = h;
                }
            }
            if (!claimed && r != kRepEmpty) hs = ((volatile unsigned long long*)t.hash)[slot];
        }
        if (kWarp) {
            r = __shfl_sync(0xffffffffu, r, 0);
            hs = __shfl_sync(0xffffffffu, hs, 0);
            claimed = __shfl_sync(0xffffffffu, claimed, 0);
        }
        if (claimed) return slot;
        if (r == kRepEmpty) return -1;
        if (hs == kHashUnset || hs == h) {
            const Str o = c.rep_str(r);
            if (o.len == s.len && bytes_equal<kWarp>(o.p, s.p, s.len, lane)) return slot;
        }
        slot = (slot + 1) & t.mask;
    }
}

template <bool kInsert>
__device__ __forceinline__ void probe_done(const Table& t, int64_t s, int64_t slot, int64_t g0, int64_t* slot_of,
                                           const int64_t* id_first, int32_t* out_ids, int64_t* out_first) {
    if (kInsert) {
        slot_of[s] = slot;
        atomicMin(&t.first[slot], (long long)(g0 + s));
        return;
    }
    const long long id = slot < 0 ? -1 : t.rep[slot];
    out_ids[s] = (int32_t)id;
    if (out_first) out_first[s] = id < 0 ? -1 : id_first[id];
}

template <bool kInsert>
__global__ void __launch_bounds__(kThreads)
vocab_probe_kernel(const int64_t* __restrict__ hdr, Table t, Chunk c, int64_t g0, const int64_t* __restrict__ totals,
                   int64_t* __restrict__ slot_of, const int64_t* __restrict__ id_first, int32_t* __restrict__ out_ids,
                   int64_t* __restrict__ out_first) {
    if (totals[0] != c.n - 1) return;           // separators do not match the string count: the host call reports it
    const int bits = (int)hdr[1];
    const int lane = threadIdx.x & 31;
    const int64_t s = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    Str str{nullptr, 0};
    if (s < c.n) str = c.str(s);
    const bool is_long = s < c.n && str.len > kShortMax;
    if (s < c.n && !is_long) {
        const uint64_t h = finish_hash(hash_thread(str.p, str.len), str.len, bits);
        probe_done<kInsert>(t, s, probe<false, kInsert>(t, c, str, h, -2 - s, lane), g0, slot_of, id_first, out_ids,
                            out_first);
    }
    __syncwarp();
    unsigned m = __ballot_sync(0xffffffffu, is_long);
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const int64_t ls = __shfl_sync(0xffffffffu, s, src);
        const Str lstr = c.str(ls);
        const uint64_t h = finish_hash(hash_warp(lstr.p, lstr.len, lane), lstr.len, bits);
        const int64_t slot = probe<true, kInsert>(t, c, lstr, h, -2 - ls, lane);
        if (lane == 0) probe_done<kInsert>(t, ls, slot, g0, slot_of, id_first, out_ids, out_first);
        __syncwarp();
    }
}

// --------------------------------------------------------------------------------------------------- scans ----
// Exclusive scan of op.value(i), i < n, in three launches (tile sums, one CTA over the tile sums, tiles again);
// op.emit(i, exclusive prefix, value) sees every item.  Values are int64 and their sum must fit.
__device__ __forceinline__ int64_t block_exclusive(int64_t v, int64_t* s_warp, int64_t* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    int64_t x = v;
    for (int d = 1; d < 32; d <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    int64_t base = 0, all = 0;
    for (int w = 0; w < n_warps; ++w) {
        base += w < warp ? s_warp[w] : 0;
        all += s_warp[w];
    }
    __syncthreads();
    *total = all;
    return base + x - v;
}

template <class Op>
__global__ void __launch_bounds__(kThreads) scan_tiles_kernel(Op op, int64_t n, int64_t* __restrict__ tile_sum) {
    __shared__ int64_t s_warp[kThreads / 32];
    const int64_t i0 = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
    int64_t acc = 0;
    for (int j = 0; j < kScanItems; ++j)
        if (i0 + j < n) acc += op.value(i0 + j);
    int64_t total;
    block_exclusive(acc, s_warp, &total);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kTopThreads)
scan_top_kernel(int64_t* __restrict__ tile_sum, int64_t n_tiles, int64_t* __restrict__ total_out) {
    __shared__ int64_t s_warp[kTopThreads / 32];
    int64_t carry = 0;
    for (int64_t b = 0; b < n_tiles; b += kTopThreads) {
        const int64_t i = b + threadIdx.x;
        const int64_t v = i < n_tiles ? tile_sum[i] : 0;
        int64_t total;
        const int64_t ex = block_exclusive(v, s_warp, &total);
        if (i < n_tiles) tile_sum[i] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) *total_out = carry;
}

template <class Op>
__global__ void __launch_bounds__(kThreads) scan_emit_kernel(Op op, int64_t n, const int64_t* __restrict__ tile_off) {
    __shared__ int64_t s_warp[kThreads / 32];
    const int64_t i0 = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
    int64_t v[kScanItems];
    int64_t acc = 0;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        v[j] = i0 + j < n ? op.value(i0 + j) : 0;
        acc += v[j];
    }
    int64_t total;
    int64_t ex = tile_off[blockIdx.x] + block_exclusive(acc, s_warp, &total);
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        if (i0 + j < n) op.emit(i0 + j, ex, v[j]);
        ex += v[j];
    }
}

// separator k (the k-th NUL) starts string k + 1
struct BoundsOp {
    const uint8_t* bytes;
    int64_t* starts;
    int64_t n;
    __device__ int64_t value(int64_t i) const { return bytes[i] == 0; }
    __device__ void emit(int64_t i, int64_t ex, int64_t v) const {
        if (v && ex + 1 < n) starts[ex + 1] = i + 1;
    }
};

// new string: (1 << 32) | its byte length, so one scan gives its rank (high word) and arena offset (low word)
struct NewOp {
    Table t;
    Chunk c;
    int64_t g0;
    const int64_t* totals;
    const int64_t* slot_of;
    int64_t* new_list;
    int64_t* new_off;
    __device__ int64_t value(int64_t s) const {
        if (totals[0] != c.n - 1 || t.first[slot_of[s]] != g0 + s) return 0;
        return (1ll << 32) | c.str(s).len;
    }
    __device__ void emit(int64_t s, int64_t ex, int64_t v) const {
        if (!v) return;
        new_list[ex >> 32] = s;
        new_off[ex >> 32] = ex & 0xffffffffll;
    }
};

template <class Op>
static int run_scan(const Op& op, int64_t n, int64_t* tile_sum, int64_t* total, cudaStream_t st) {
    if (n == 0) {
        EZR_CUDA(cudaMemsetAsync(total, 0, sizeof(int64_t), st));
        return EZR_OK;
    }
    const int64_t tiles = (n + kScanTile - 1) / kScanTile;
    scan_tiles_kernel<Op><<<(unsigned)tiles, kThreads, 0, st>>>(op, n, tile_sum);
    EZR_LAUNCH_CHECK();
    scan_top_kernel<<<1, kTopThreads, 0, st>>>(tile_sum, tiles, total);
    EZR_LAUNCH_CHECK();
    scan_emit_kernel<Op><<<(unsigned)tiles, kThreads, 0, st>>>(op, n, tile_sum);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

// -------------------------------------------------------------------------------------------- maintenance ----
__global__ void vocab_fill_kernel(int64_t* __restrict__ hdr, Table t, int64_t cap, int bits,
                                  const int64_t* __restrict__ bits_from) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) {
        hdr[0] = cap;
        hdr[1] = bits_from ? bits_from[1] : bits;
    }
    if (i < cap) {
        t.rep[i] = kRepEmpty;
        t.hash[i] = kHashUnset;
        t.first[i] = LLONG_MAX;
    }
}

// every slot of a table between calls holds an id with its hash: re-placed by that hash, no comparisons needed
__global__ void vocab_rehash_kernel(Table from, int64_t cap_from, Table to) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap_from) return;
    const long long r = from.rep[i];
    if (r < 0) return;
    const unsigned long long h = from.hash[i];
    int64_t slot = slot_start(h, to.mask);
    while (atomicCAS((unsigned long long*)&to.rep[slot], (unsigned long long)kRepEmpty, (unsigned long long)r) !=
           (unsigned long long)kRepEmpty)
        slot = (slot + 1) & to.mask;
    to.hash[slot] = h;
    to.first[slot] = from.first[i];
}

// a chunk that cannot be published: its claims are undone.  Slots claimed in the chunk were empty when every older
// slot was placed, so no older probe sequence passes through them and emptying them restores the table.
__global__ void vocab_rollback_kernel(Table t, int64_t cap) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < cap && t.rep[i] <= -2) {
        t.rep[i] = kRepEmpty;
        t.hash[i] = kHashUnset;
        t.first[i] = LLONG_MAX;
    }
}

__global__ void __launch_bounds__(kThreads)
vocab_publish_kernel(Table t, Chunk c, int64_t g0, int64_t n_new, int64_t n_ids, int64_t arena_used,
                     const int64_t* __restrict__ slot_of, const int64_t* __restrict__ new_list,
                     const int64_t* __restrict__ new_off, int64_t* __restrict__ id_first, int64_t* __restrict__ arena_off) {
    const int64_t r = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (r >= n_new) return;
    const int64_t s = new_list[r], id = n_ids + r;
    t.rep[slot_of[s]] = id;
    id_first[id] = g0 + s;
    arena_off[id + 1] = arena_used + new_off[r] + c.str(s).len;
}

// one warp per new string
__global__ void __launch_bounds__(kThreads)
vocab_copy_kernel(Chunk c, int64_t n_new, int64_t arena_used, const int64_t* __restrict__ new_list,
                  const int64_t* __restrict__ new_off, uint8_t* __restrict__ arena) {
    const int64_t r = ((int64_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
    if (r >= n_new) return;
    const Str s = c.str(new_list[r]);
    uint8_t* dst = arena + arena_used + new_off[r];
    for (int64_t i = threadIdx.x & 31; i < s.len; i += 32) dst[i] = s.p[i];
}

__global__ void __launch_bounds__(kThreads)
vocab_map_kernel(Table t, int64_t n, const int64_t* __restrict__ slot_of, const int64_t* __restrict__ id_first,
                 int32_t* __restrict__ out_ids, int64_t* __restrict__ out_first) {
    const int64_t s = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (s >= n) return;
    const long long id = t.rep[slot_of[s]];
    out_ids[s] = (int32_t)id;
    if (out_first) out_first[s] = id_first[id];
}

// ---------------------------------------------------------------------------------------------- workspace ----
struct Ws {
    int64_t* starts;
    int64_t* slot_of;
    int64_t* new_list;
    int64_t* new_off;
    int64_t* tiles;
    int64_t* totals;     // [0] separators, [1] (new strings << 32) | new bytes
};

static size_t ws_layout(int64_t n, int64_t n_bytes, void* base, Ws* w) {
    const int64_t tiles = (std::max(n, n_bytes) + kScanTile - 1) / kScanTile;
    size_t off = 0;
    int64_t** parts[] = {&w->starts, &w->slot_of, &w->new_list, &w->new_off, &w->tiles, &w->totals};
    const int64_t sizes[] = {n, n, n, n, tiles, 4};
    for (int i = 0; i < 6; ++i) {
        if (base) *parts[i] = (int64_t*)((char*)base + off);
        off += align_up((size_t)std::max<int64_t>(sizes[i], 1) * sizeof(int64_t), 256);
    }
    return off;
}

static inline unsigned grid_of(int64_t n, int per) { return (unsigned)std::max<int64_t>((n + per - 1) / per, 1); }

static int check_table_cap(int64_t cap) {
    EZR_CHECK_ARG(cap >= 2 && cap <= (1ll << 40) && (cap & (cap - 1)) == 0,
                  "vocab: table capacity %lld must be a power of two in [2, 2^40]", (long long)cap);
    return EZR_OK;
}

static int bounds(const uint8_t* bytes, int64_t n_bytes, int64_t n, const Ws& w, cudaStream_t st) {
    EZR_CUDA(cudaMemsetAsync(w.starts, 0, sizeof(int64_t), st));
    return run_scan(BoundsOp{bytes, w.starts, n}, n_bytes, w.tiles, &w.totals[0], st);
}

}  // namespace ezr

using namespace ezr;

extern "C" {

int ezr_vocab_set_hash_bits(int32_t bits) {
    EZR_CHECK_ARG(bits >= 1 && bits <= 64, "vocab_set_hash_bits: %d outside [1, 64]", bits);
    g_vocab_bits = bits;
    return EZR_OK;
}

size_t ezr_vocab_table_bytes(int64_t capacity) {
    return capacity < 0 ? 0 : (size_t)(kHdr + 3 * capacity) * sizeof(int64_t);
}

size_t ezr_vocab_workspace(int64_t n_strings, int64_t n_bytes) {
    Ws w;
    return ws_layout(std::max<int64_t>(n_strings, 0), std::max<int64_t>(n_bytes, 0), nullptr, &w);
}

int ezr_vocab_table_init(void* table, int64_t capacity, void* stream) {
    if (int rc = check_table_cap(capacity)) return rc;
    EZR_CHECK_ARG(table, "vocab_table_init: NULL table");
    vocab_fill_kernel<<<grid_of(capacity, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
        (int64_t*)table, Table(table, capacity), capacity, g_vocab_bits, nullptr);
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_vocab_table_grow(const void* table, int64_t capacity, void* new_table, int64_t new_capacity, void* stream) {
    if (int rc = check_table_cap(capacity)) return rc;
    if (int rc = check_table_cap(new_capacity)) return rc;
    EZR_CHECK_ARG(table && new_table && table != new_table, "vocab_table_grow: NULL or identical tables");
    EZR_CHECK_ARG(new_capacity >= capacity, "vocab_table_grow: %lld slots cannot hold a table of %lld",
                  (long long)new_capacity, (long long)capacity);
    cudaStream_t st = (cudaStream_t)stream;
    vocab_fill_kernel<<<grid_of(new_capacity, kThreads), kThreads, 0, st>>>(
        (int64_t*)new_table, Table(new_table, new_capacity), new_capacity, 0, (const int64_t*)table);
    EZR_LAUNCH_CHECK();
    vocab_rehash_kernel<<<grid_of(capacity, kThreads), kThreads, 0, st>>>(
        Table((void*)table, capacity), capacity, Table(new_table, new_capacity));
    EZR_LAUNCH_CHECK();
    return EZR_OK;
}

int ezr_vocab_insert(void* table, int64_t capacity, const uint8_t* bytes, int64_t n_bytes, int64_t n_strings,
                     int64_t first_index, uint8_t* arena, int64_t arena_capacity, int64_t* arena_off,
                     int64_t* id_first, int64_t id_capacity, int64_t* state_host, int32_t* out_ids,
                     int64_t* out_first, void* workspace, size_t ws_bytes, void* stream) {
    if (int rc = check_table_cap(capacity)) return rc;
    EZR_CHECK_ARG(n_strings >= 0 && n_bytes >= 0 && n_bytes <= kMaxChunkBytes && first_index >= 0,
                  "vocab_insert: n_strings=%lld / n_bytes=%lld (at most 2^32 - 1) / first_index=%lld",
                  (long long)n_strings, (long long)n_bytes, (long long)first_index);
    EZR_CHECK_ARG(n_strings > 0 || n_bytes == 0, "vocab_insert: bytes without strings");
    if (n_strings == 0) return EZR_OK;
    EZR_CHECK_ARG(table && arena_off && id_first && state_host && out_ids && workspace && (bytes || n_bytes == 0),
                  "vocab_insert: NULL argument");
    const int64_t n_ids = state_host[0], arena_used = state_host[1];
    EZR_CHECK_ARG(n_ids >= 0 && arena_used >= 0, "vocab_insert: bad state");
    if (2 * (n_ids + n_strings) > capacity) {
        set_error("vocab_insert: %lld ids + %lld strings pass the load limit 1/2 of %lld slots: grow the table first",
                  (long long)n_ids, (long long)n_strings, (long long)capacity);
        return EZR_ERR_WORKSPACE;
    }
    Ws w;
    if (ws_bytes < ws_layout(n_strings, n_bytes, workspace, &w)) {
        set_error("vocab_insert: workspace of %zu bytes, %zu needed", ws_bytes, ezr_vocab_workspace(n_strings, n_bytes));
        return EZR_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const Table t(table, capacity);
    const Chunk c{bytes, w.starts, n_strings, n_bytes, arena, arena_off};
    if (int rc = bounds(bytes, n_bytes, n_strings, w, st)) return rc;
    vocab_probe_kernel<true><<<grid_of(n_strings, kThreads), kThreads, 0, st>>>(
        (const int64_t*)table, t, c, first_index, w.totals, w.slot_of, nullptr, nullptr, nullptr);
    EZR_LAUNCH_CHECK();
    if (int rc = run_scan(NewOp{t, c, first_index, w.totals, w.slot_of, w.new_list, w.new_off}, n_strings, w.tiles,
                          &w.totals[1], st))
        return rc;
    int64_t tot[2];
    EZR_CUDA(cudaMemcpyAsync(tot, w.totals, sizeof(tot), cudaMemcpyDeviceToHost, st));
    EZR_CUDA(cudaStreamSynchronize(st));
    if (tot[0] != n_strings - 1) {
        set_error("vocab_insert: %lld NUL separators for %lld strings (a string contains NUL?)", (long long)tot[0],
                  (long long)n_strings);
        return EZR_ERR_INVALID;
    }
    const int64_t n_new = tot[1] >> 32, new_bytes = tot[1] & 0xffffffffll;
    const bool id_overflow = n_ids + n_new > INT32_MAX;
    if (id_overflow || n_ids + n_new > id_capacity || arena_used + new_bytes > arena_capacity) {
        vocab_rollback_kernel<<<grid_of(capacity, kThreads), kThreads, 0, st>>>(t, capacity);
        EZR_LAUNCH_CHECK();
        EZR_CUDA(cudaStreamSynchronize(st));
        if (id_overflow) {
            set_error("vocab_insert: %lld + %lld ids overflow int32", (long long)n_ids, (long long)n_new);
            return EZR_ERR_INVALID;
        }
        set_error("vocab_insert: %lld new strings / %lld new bytes do not fit the id capacity %lld / arena %lld",
                  (long long)n_new, (long long)new_bytes, (long long)id_capacity, (long long)arena_capacity);
        return EZR_ERR_WORKSPACE;
    }
    if (n_new > 0) {
        vocab_publish_kernel<<<grid_of(n_new, kThreads), kThreads, 0, st>>>(
            t, c, first_index, n_new, n_ids, arena_used, w.slot_of, w.new_list, w.new_off, id_first, arena_off);
        EZR_LAUNCH_CHECK();
        vocab_copy_kernel<<<grid_of(n_new, kThreads / 32), kThreads, 0, st>>>(c, n_new, arena_used, w.new_list,
                                                                              w.new_off, arena);
        EZR_LAUNCH_CHECK();
    }
    vocab_map_kernel<<<grid_of(n_strings, kThreads), kThreads, 0, st>>>(t, n_strings, w.slot_of, id_first, out_ids,
                                                                        out_first);
    EZR_LAUNCH_CHECK();
    state_host[0] = n_ids + n_new;
    state_host[1] = arena_used + new_bytes;
    return EZR_OK;
}

int ezr_vocab_lookup(const void* table, int64_t capacity, const uint8_t* bytes, int64_t n_bytes, int64_t n_strings,
                     const uint8_t* arena, const int64_t* arena_off, const int64_t* id_first, int32_t* out_ids,
                     int64_t* out_first, void* workspace, size_t ws_bytes, void* stream) {
    if (int rc = check_table_cap(capacity)) return rc;
    EZR_CHECK_ARG(n_strings >= 0 && n_bytes >= 0 && n_bytes <= kMaxChunkBytes,
                  "vocab_lookup: n_strings=%lld / n_bytes=%lld (at most 2^32 - 1)", (long long)n_strings,
                  (long long)n_bytes);
    EZR_CHECK_ARG(n_strings > 0 || n_bytes == 0, "vocab_lookup: bytes without strings");
    if (n_strings == 0) return EZR_OK;
    EZR_CHECK_ARG(table && arena_off && id_first && out_ids && workspace && (bytes || n_bytes == 0),
                  "vocab_lookup: NULL argument");
    Ws w;
    if (ws_bytes < ws_layout(n_strings, n_bytes, workspace, &w)) {
        set_error("vocab_lookup: workspace of %zu bytes, %zu needed", ws_bytes, ezr_vocab_workspace(n_strings, n_bytes));
        return EZR_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const Chunk c{bytes, w.starts, n_strings, n_bytes, arena, arena_off};
    if (int rc = bounds(bytes, n_bytes, n_strings, w, st)) return rc;
    vocab_probe_kernel<false><<<grid_of(n_strings, kThreads), kThreads, 0, st>>>(
        (const int64_t*)table, Table((void*)table, capacity), c, 0, w.totals, nullptr, id_first, out_ids, out_first);
    EZR_LAUNCH_CHECK();
    int64_t seps;
    EZR_CUDA(cudaMemcpyAsync(&seps, w.totals, sizeof(seps), cudaMemcpyDeviceToHost, st));
    EZR_CUDA(cudaStreamSynchronize(st));
    if (seps != n_strings - 1) {
        set_error("vocab_lookup: %lld NUL separators for %lld strings (a string contains NUL?)", (long long)seps,
                  (long long)n_strings);
        return EZR_ERR_INVALID;
    }
    return EZR_OK;
}

int ezr_vocab_read(const uint8_t* arena, const int64_t* arena_off, int64_t id_lo, int64_t id_hi,
                   uint8_t* bytes_host, size_t bytes_cap, int64_t* off_host, void* stream) {
    EZR_CHECK_ARG(arena_off && off_host && 0 <= id_lo && id_lo <= id_hi, "vocab_read: NULL argument or bad id range");
    cudaStream_t st = (cudaStream_t)stream;
    EZR_CUDA(cudaMemcpyAsync(off_host, arena_off + id_lo, (size_t)(id_hi - id_lo + 1) * sizeof(int64_t),
                             cudaMemcpyDeviceToHost, st));
    EZR_CUDA(cudaStreamSynchronize(st));
    const int64_t nb = off_host[id_hi - id_lo] - off_host[0];
    EZR_CHECK_ARG(nb >= 0 && (size_t)nb <= bytes_cap && (bytes_host || nb == 0),
                  "vocab_read: %lld bytes do not fit %zu", (long long)nb, bytes_cap);
    if (nb > 0) {
        EZR_CUDA(cudaMemcpyAsync(bytes_host, arena + off_host[0], (size_t)nb, cudaMemcpyDeviceToHost, st));
        EZR_CUDA(cudaStreamSynchronize(st));
    }
    return EZR_OK;
}

}  // extern "C"
