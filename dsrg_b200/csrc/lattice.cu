// Permutohedral lattice construction on the GPU (sm_90a).
//
// Replaces Permutohedral::init + HashTable (CRF/src/permutohedral.cpp:54-131, :140-321) and
// DenseKernel::initLattice (CRF/src/pairwise.cpp:40-62) of the reference, for a whole batch at
// once.  The arithmetic that decides WHICH simplex a pixel falls into follows the reference's
// SSE code path operation by operation (round-to-nearest-even, no FMA contraction: every float
// op is an explicit __f*_rn intrinsic); the hash table itself is a GPU design (64-bit packed
// keys, CAS insertion).
//
// Vertex numbering does not change the filter's values, but it decides the blur's memory traffic: a blur pass
// reads 3 to 27 rows per output row through the neighbour table.  Insertion hands out ids in arrival order, which
// with all of an image's insert blocks in flight at once scatters neighbouring vertices over a buffer larger than
// the L2.  So the build renumbers every lattice (k_renum_*): a vertex's key is its first incidence in tile-major
// pixel order (tile, pixel's thread index in the tile, r; tiles.cu's geometry), and the ids are the ranks of the
// keys.  Lattice neighbours then sit a few ids apart for the spatial lattice and mostly so for the bilateral one,
// each tile's rows are a few contiguous runs, and the numbering is deterministic.
#include "common.cuh"
#include "simplex.cuh"

namespace dsrg {

// ---------------------------------------------------------------------------------------------
// packed keys: d=2 -> 2 x 16 bit (exactly the reference's `short`), d=5 -> 5 x 12 bit
// ---------------------------------------------------------------------------------------------
template <int D>
struct KeyBits {
    static constexpr int bits = (D == 2) ? 16 : 12;
    static constexpr int lo = -(1 << (bits - 1));
    static constexpr int hi = (1 << (bits - 1)) - 1;
};

template <int D>
__device__ __forceinline__ uint64_t pack_key(const int *key) {
    constexpr int BITS = KeyBits<D>::bits;
    uint64_t k = 0;
#pragma unroll
    for (int i = 0; i < D; i++) k |= (uint64_t)((uint32_t)key[i] & ((1u << BITS) - 1)) << (i * BITS);
    return k;
}

template <int D>
__device__ __forceinline__ void unpack_key(uint64_t k, int *key) {
    constexpr int BITS = KeyBits<D>::bits;
#pragma unroll
    for (int i = 0; i < D; i++) {
        int v = (int)((k >> (i * BITS)) & ((1u << BITS) - 1));
        key[i] = (v << (32 - BITS)) >> (32 - BITS);  // sign extend
    }
}

__device__ __forceinline__ uint32_t hash_slot(uint64_t k, uint32_t cap) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return (uint32_t)(((k >> 32) * (uint64_t)cap) >> 32);
}

__device__ __forceinline__ uint64_t ld_relaxed_u64(const uint64_t *p) {
    uint64_t v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
    return v;
}

// insert-or-find; the winner of an empty slot allocates the next vertex id of its image (in arrival order: the
// renumbering replaces it before anything else reads it)
__device__ __forceinline__ int hash_insert(uint64_t *keys, int32_t *hval, int32_t *vslot,
                                           int32_t *vcount, uint32_t cap, uint64_t k) {
    uint32_t s = hash_slot(k, cap);
    while (true) {
        uint64_t cur = ld_relaxed_u64(keys + s);
        if (cur == k) return (int)s;
        if (cur == kEmptyKey) {
            unsigned long long old =
                atomicCAS((unsigned long long *)(keys + s), (unsigned long long)kEmptyKey,
                          (unsigned long long)k);
            if (old == kEmptyKey) {
                int id = atomicAdd(vcount, 1);
                vslot[id] = (int)s;
                asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(hval + s), "r"(id) : "memory");
                return (int)s;
            }
            if (old == k) return (int)s;
        }
        s = (s + 1 == cap) ? 0 : s + 1;
    }
}

__device__ __forceinline__ int hash_lookup(const uint64_t *keys, uint32_t cap, uint64_t k) {
    uint32_t s = hash_slot(k, cap);
    while (true) {
        uint64_t cur = keys[s];
        if (cur == k) return (int)s;
        if (cur == kEmptyKey) return -1;
        s = (s + 1 == cap) ? 0 : s + 1;
    }
}

struct BuildArgs {
    int N, P, W;
    int tile_w, tiles_x, ntiles;
    uint32_t cap;
    int capv;
    float sigma[5];
    float scale[5];
    const uint8_t *image;  // [B][N][3] or nullptr
    int32_t *off;
    float *bary;
    uint64_t *hkeys;
    int32_t *hval, *aslot, *vcount, *vkey;
    int *err;
    const float *feat;  // k_lattice_insert<kFeatLattice>: the caller's features [B][5][N]
    int *bad;           // ... and its per-image key-range flags [B]
};

// A pixel's position in tile-major order (tiles.cu: tile index, then the pixel's thread index in the tile); the
// phantom lanes all sit at position ntiles * kTileThreads, after every pixel.  Renumbering key of incidence
// (pixel, r): pos * (d+1) + r.
__device__ __forceinline__ int tile_major_pos(int x, int y, int tile_w, int tiles_x) {
    const int tx = x / tile_w, ty = y / kTileH;
    return (ty * tiles_x + tx) * kTileThreads + (y - ty * kTileH) * kTileW + (x - tx * tile_w);
}

// ---------------------------------------------------------------------------------------------
// Kernel 1: one thread per pixel (plus the phantom tail lanes): features -> elevate -> simplex ->
// rank -> barycentric -> d+1 vertex keys -> hash insert.  Follows permutohedral.cpp:191-276.
// D = kFeatLattice: the bilateral lattice (d = 5) on the caller's features (a.feat [B][5][N], taken as they are), and a
// key outside the packed range flags the image in a.bad[b] instead of the engine's error flag.
// ---------------------------------------------------------------------------------------------
constexpr int kFeatLattice = -5;

template <int D>
__global__ void __launch_bounds__(kThreads) k_lattice_insert(BuildArgs a) {
    constexpr bool FEAT = D == kFeatLattice;
    constexpr int DIM = FEAT ? 5 : D;
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool valid = i < a.N + a.P;
    const bool real = i < a.N;

    float f[DIM];
#pragma unroll
    for (int j = 0; j < DIM; j++) f[j] = 0.0f;  // phantom lanes carry feature 0 (:196)
    int pos = a.ntiles * kTileThreads;
    if (real) {
        const int x = i % a.W, y = i / a.W;
        pos = tile_major_pos(x, y, a.tile_w, a.tiles_x);
        if constexpr (FEAT) {
#pragma unroll
            for (int j = 0; j < DIM; j++) f[j] = __ldg(a.feat + ((size_t)b * DIM + j) * a.N + i);
        } else {
            lattice_features<DIM>(x, y, a.image, b, a.N, i, a.sigma, f);
        }
    }
    // elevate, simplex, rank (simplex.cuh)
    float el[DIM + 1], rem0[DIM + 1];
    int rank[DIM + 1];
    lattice_simplex<DIM>(f, a.scale, el, rem0, rank);
    const float inv = __fdiv_rn(1.0f, (float)(DIM + 1));
    // barycentric (:245-263), same accumulation order as the reference
    float bc[DIM + 2];
#pragma unroll
    for (int q = 0; q <= DIM + 1; q++) bc[q] = 0.0f;
#pragma unroll
    for (int k = 0; k <= DIM; k++) {
        float v = __fmul_rn(__fsub_rn(el[k], rem0[k]), inv);
        int p = DIM - rank[k];
#pragma unroll
        for (int q = 0; q <= DIM + 1; q++) {
            if (q == p) bc[q] = __fadd_rn(bc[q], v);
            if (q == p + 1) bc[q] = __fsub_rn(bc[q], v);
        }
    }
    bc[0] = __fadd_rn(bc[0], __fadd_rn(1.0f, bc[DIM + 1]));

    // vertices (:268-275)
    uint64_t *keys = a.hkeys + (size_t)b * a.cap;
    int32_t *hval = a.hval + (size_t)b * a.cap;
    int32_t *aslot = a.aslot + (size_t)b * a.capv;
    int32_t *vkey = a.vkey + (size_t)b * a.capv;
    int32_t *vcount = a.vcount + b;
    const unsigned lane = threadIdx.x & 31;
    bool range_bad = false;
#pragma unroll
    for (int r = 0; r <= DIM; r++) {
        int key[DIM];
#pragma unroll
        for (int k = 0; k < DIM; k++) {
            int canon = (rank[k] <= DIM - r) ? r : r - (DIM + 1);  // canonical simplex (:171-176)
            key[k] = (int)rem0[k] + canon;
            if (key[k] < KeyBits<DIM>::lo || key[k] > KeyBits<DIM>::hi) range_bad = true;
        }
        uint64_t pk = pack_key<DIM>(key);
        // neighbouring pixels mostly share vertices: one insert per distinct key per warp
        unsigned peers = __match_any_sync(0xffffffffu, valid ? pk : (kEmptyKey - 1 - lane));
        int leader = __ffs(peers) - 1;
        int id = 0;
        // the first incidence of the vertex among the lanes, for the renumbering key (vkey is kNoKey between builds)
        const int kmin = __reduce_min_sync(peers, valid ? pos * (DIM + 1) + r : kNoKey);
        if (valid && (int)lane == leader) {
            const int slot = hash_insert(keys, hval, aslot, vcount, a.cap, pk);
            // the slot's owner publishes the vertex id right after winning the CAS; owners of the
            // same key always sit in other warps (one leader per key per warp), so this cannot
            // wait on a lane of the same warp
            do {
                asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(id) : "l"(hval + slot) : "memory");
            } while (id < 0);
            atomicMin(vkey + id, kmin);
        }
        id = __shfl_sync(0xffffffffu, id, leader);
        if (real) {
            size_t at = ((size_t)b * (DIM + 1) + r) * a.N + i;
            a.off[at] = id + 1;  // local row (row 0 of every image is its zero row)
            a.bary[at] = bc[r];
        }
    }
    if constexpr (FEAT) {
        if (valid && range_bad) a.bad[b] = 1;
    } else {
        if (valid && range_bad) *a.err = DSRG_E_KEYRANGE;
    }
}

// rowbase[b] = first value row of image b (its zero row); rowbase[B] = total rows
__global__ void k_rowbase(const int32_t *vcount, int32_t *rowbase, int B, int shared) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        int acc = 0;
        for (int b = 0; b <= B; b++) {
            rowbase[b] = acc;
            if (b < B) acc += vcount[shared ? 0 : b] + 1;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Renumbering: new id = rank of the vertex's key (vkey, its first incidence, from k_lattice_insert) among its
// image's keys.  The keys are marked in a bitmap over the key space (one bit per (pixel, r)); the rank of a key is
// the number of marked bits before it: a per-chunk prefix (k_renum_scan, words of 32 bits, kRenumChunk words per
// chunk), a per-image prefix over the chunks (k_renum_chunks) and the popcount inside the word.
// ---------------------------------------------------------------------------------------------
// words of the key-space bitmap per image (a whole number of chunks)
long long renum_words(int ntiles, int dp1) {
    const long long keys = ((long long)ntiles * kTileThreads + 1) * dp1;
    return (keys + 32LL * kRenumChunk - 1) / (32LL * kRenumChunk) * kRenumChunk;
}

__global__ void __launch_bounds__(kThreads)
k_renum_mark(const int32_t *vcount, const int32_t *vkey, uint2 *words, int capv, long long nwords) {
    const int b = blockIdx.y;
    const int V = vcount[b];
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) {
        const int k = vkey[(size_t)b * capv + v];
        atomicOr(&words[b * nwords + (k >> 5)].x, 1u << (k & 31));
    }
}

// exclusive block-wide scan of one value per thread (kThreads threads); *total gets the block's sum
__device__ __forceinline__ int block_exclusive_scan(int v, int *total) {
    __shared__ int wsum[kThreads / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += n;
    }
    if (lane == 31) wsum[wid] = incl;
    __syncthreads();
    int base = 0, all = 0;
#pragma unroll
    for (int k = 0; k < kThreads / 32; k++) {
        base += k < wid ? wsum[k] : 0;
        all += wsum[k];
    }
    __syncthreads();  // wsum may be reused by the next call
    *total = all;
    return base + incl - v;
}

// per word: the marked bits before it inside its chunk (.y); per chunk: its marked bits
__global__ void __launch_bounds__(kThreads) k_renum_scan(uint2 *words, int32_t *chunk_sum, long long nwords, int nchunks) {
    const int b = blockIdx.y, c = blockIdx.x;
    uint2 *w = words + b * nwords + (long long)c * kRenumChunk + 4 * threadIdx.x;
    int n[4], s = 0;
#pragma unroll
    for (int q = 0; q < 4; q++) s += n[q] = __popc(w[q].x);
    int total;
    int pre = block_exclusive_scan(s, &total);
#pragma unroll
    for (int q = 0; q < 4; q++) {
        w[q].y = (uint32_t)pre;
        pre += n[q];
    }
    if (threadIdx.x == 0) chunk_sum[(size_t)b * nchunks + c] = total;
}

// per image: chunk sums -> exclusive prefix
__global__ void __launch_bounds__(kThreads) k_renum_chunks(int32_t *chunk_sum, int nchunks) {
    int32_t *cs = chunk_sum + (size_t)blockIdx.x * nchunks;
    int carry = 0;
    for (int c0 = 0; c0 < nchunks; c0 += kThreads) {
        const int c = c0 + threadIdx.x;
        const int v = c < nchunks ? cs[c] : 0;
        int total;
        const int pre = block_exclusive_scan(v, &total);
        if (c < nchunks) cs[c] = carry + pre;
        carry += total;
    }
}

// old id v -> new id: vkey[v] becomes the new id (k_norm_splat rewrites off with it), hval and vslot follow the new
// numbering
__global__ void __launch_bounds__(kThreads)
k_renum_rank(const int32_t *vcount, int32_t *vkey, const uint2 *words, const int32_t *chunk_sum, const int32_t *aslot,
             int32_t *hval, int32_t *vslot, uint32_t cap, int capv, long long nwords, int nchunks) {
    const int b = blockIdx.y;
    const int V = vcount[b];
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) {
        const size_t at = (size_t)b * capv + v;
        const int k = vkey[at];
        const uint2 w = words[b * nwords + (k >> 5)];
        const int id = chunk_sum[(size_t)b * nchunks + (k >> 5) / kRenumChunk] + (int)w.y +
                       __popc(w.x & ((1u << (k & 31)) - 1u));
        vkey[at] = id;
        const int slot = aslot[at];
        hval[(size_t)b * cap + slot] = id;
        vslot[(size_t)b * capv + id] = slot;
    }
}

// Kernel 3: blur neighbours of every vertex (:305-318).  Missing neighbour -> the zero row.
template <int D>
__global__ void __launch_bounds__(kThreads)
k_lattice_neighbors(const uint64_t *hkeys, const int32_t *hval, const int32_t *vslot,
                    const int32_t *vcount, const int32_t *rowbase, int2 *nbr, long long nbr_stride,
                    uint32_t cap, int capv, int shared) {
    const int b = blockIdx.y;
    const int V = vcount[b];
    const long long base = shared ? 0 : rowbase[b];
    const uint64_t *keys = hkeys + (size_t)b * cap;
    const int32_t *hv = hval + (size_t)b * cap;
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v <= V; v += gridDim.x * blockDim.x) {
        if (v == V) {  // the zero row points at itself so that blurring keeps it at zero
#pragma unroll
            for (int j = 0; j <= D; j++) nbr[(size_t)j * nbr_stride + base] = make_int2((int)base, (int)base);
            continue;
        }
        int key[D];
        unpack_key<D>(keys[vslot[(size_t)b * capv + v]], key);
        const long long row = base + 1 + v;
#pragma unroll
        for (int j = 0; j <= D; j++) {
            int n1[D], n2[D];
            bool ok1 = true, ok2 = true;
#pragma unroll
            for (int k = 0; k < D; k++) {
                n1[k] = key[k] - 1;
                n2[k] = key[k] + 1;
                if (k == j) {
                    n1[k] = key[k] + D;
                    n2[k] = key[k] - D;
                }
                ok1 &= (n1[k] >= KeyBits<D>::lo && n1[k] <= KeyBits<D>::hi);
                ok2 &= (n2[k] >= KeyBits<D>::lo && n2[k] <= KeyBits<D>::hi);
            }
            int s1 = ok1 ? hash_lookup(keys, cap, pack_key<D>(n1)) : -1;
            int s2 = ok2 ? hash_lookup(keys, cap, pack_key<D>(n2)) : -1;
            int r1 = s1 < 0 ? (int)base : (int)(base + 1 + hv[s1]);
            int r2 = s2 < 0 ? (int)base : (int)(base + 1 + hv[s2]);
            nbr[(size_t)j * nbr_stride + row] = make_int2(r1, r2);
        }
    }
}

// Kernel 4: give the slots back (the tables stay all-empty between batches, no big memset)
__global__ void __launch_bounds__(kThreads)
k_lattice_cleanup(uint64_t *hkeys, int32_t *hval, const int32_t *vslot, const int32_t *vcount, uint32_t cap,
                  int capv) {
    const int b = blockIdx.y;
    const int V = vcount[b];
    for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) {
        const size_t at = (size_t)b * cap + vslot[(size_t)b * capv + v];
        hkeys[at] = kEmptyKey;
        hval[at] = -1;
    }
}

// ---------------------------------------------------------------------------------------------
// Normalisation: norm = 1/sqrt(K 1 + 1e-20), pairwise.cpp:44,54-57, with K 1 evaluated like
// Permutohedral::seqCompute(value_size=1) (permutohedral.cpp:476-527).
// ---------------------------------------------------------------------------------------------
// also finishes the renumbering: off still holds arrival-order ids, vkey maps them to the new ones (k_renum_rank)
__global__ void __launch_bounds__(kThreads)
k_norm_splat(int32_t *off, const float *bary, const int32_t *rowbase, const int32_t *vkey, float *nv, int N,
             int dp1, int capv) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int base = rowbase[b];
    const int32_t *perm = vkey + (size_t)b * capv;
    for (int r = 0; r < dp1; r++) {
        size_t at = ((size_t)b * dp1 + r) * N + i;
        const int row = perm[off[at] - 1] + 1;
        off[at] = row;
        atomicAdd(nv + base + row, bary[at]);  // values[o] += w * 1 (:491)
    }
}

__global__ void __launch_bounds__(kThreads)
k_norm_blur(const float *in, float *out, const int2 *nbr, const int32_t *rowbase, int B) {
    const int rows = rowbase[B];
    for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < rows; g += gridDim.x * blockDim.x) {
        int2 n = nbr[g];
        // (float)(old + 0.5*(n1+n2)) evaluated in double (:505) == this single-rounding float form
        out[g] = __fadd_rn(in[g], __fmul_rn(0.5f, __fadd_rn(in[n.x], in[n.y])));
    }
}

// also resets the renumbering keys for the next build (vkey is kNoKey between builds; k_norm_splat was its last reader)
__global__ void __launch_bounds__(kThreads)
k_norm_slice(const int32_t *off, const float *bary, const int32_t *rowbase, const float *nv,
             float *norm, int N, int dp1, float alpha, int32_t *vkey, const int32_t *vcount, int capv) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    for (int v = i, V = vcount[b]; v < V; v += N) vkey[(size_t)b * capv + v] = kNoKey;
    const int base = rowbase[b];
    float acc = 0.0f;
    for (int r = 0; r < dp1; r++) {
        size_t at = ((size_t)b * dp1 + r) * N + i;
        float w = bary[at];
        // out += w * values[o] * alpha (:520)
        acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(w, nv[base + off[at]]), alpha));
    }
    norm[(size_t)b * N + i] = (float)(1.0 / sqrt((double)acc + 1e-20));  // pairwise.cpp:56
}

template <int D>
static int build_impl(Engine *e, Lattice &L, int nb, const uint8_t *image, const float *feat, int *bad,
                      cudaStream_t s) {
    BuildArgs a;
    a.N = L.N;
    a.P = L.P;
    a.W = e->W;
    a.tile_w = e->tile_w;
    a.tiles_x = e->tiles_x;
    a.ntiles = e->ntiles;
    a.cap = (uint32_t)L.cap;
    a.capv = L.capv;
    for (int i = 0; i < 5; i++) {
        a.sigma[i] = L.sigma[i];
        a.scale[i] = L.scale[i];
    }
    a.image = image;
    a.off = L.off;
    a.bary = L.bary;
    a.hkeys = L.hkeys;
    a.hval = L.hval;
    a.aslot = L.aslot;
    a.vcount = L.vcount;
    a.vkey = L.vkey;
    a.err = e->dev_err;
    a.feat = feat;
    a.bad = bad;
    DSRG_CUDA_TRY(cudaMemsetAsync(L.vcount, 0, sizeof(int32_t) * nb, s));
    const long long nwords = renum_words(e->ntiles, D + 1);
    const int nchunks = (int)(nwords / kRenumChunk);
    DSRG_CUDA_TRY(cudaMemsetAsync(L.rn_words, 0, sizeof(uint2) * nb * nwords, s));
    dim3 gp(cdiv(L.N + L.P, kThreads), nb);
    if (feat) {
        DSRG_CUDA_TRY(cudaMemsetAsync(bad, 0, sizeof(int) * nb, s));
        DSRG_LAUNCH(e, T_LAT_INSERT, s, k_lattice_insert<kFeatLattice><<<gp, kThreads, 0, s>>>(a));
    } else {
        DSRG_LAUNCH(e, T_LAT_INSERT, s, k_lattice_insert<D><<<gp, kThreads, 0, s>>>(a));
    }
    DSRG_LAUNCH(e, T_LAT_MISC, s, k_rowbase<<<1, 32, 0, s>>>(L.vcount, L.rowbase, L.shared ? e->maxB : nb, L.shared));
    dim3 gv(2 * e->sm_count, nb);
    DSRG_LAUNCH(e, T_LAT_MISC, s, k_renum_mark<<<gv, kThreads, 0, s>>>(L.vcount, L.vkey, L.rn_words, L.capv, nwords));
    DSRG_LAUNCH(e, T_LAT_MISC, s, k_renum_scan<<<dim3(nchunks, nb), kThreads, 0, s>>>(L.rn_words, L.rn_chunk, nwords, nchunks));
    DSRG_LAUNCH(e, T_LAT_MISC, s, k_renum_chunks<<<nb, kThreads, 0, s>>>(L.rn_chunk, nchunks));
    DSRG_LAUNCH(e, T_LAT_MISC, s,
                k_renum_rank<<<gv, kThreads, 0, s>>>(L.vcount, L.vkey, L.rn_words, L.rn_chunk, L.aslot, L.hval, L.vslot,
                                                     a.cap, L.capv, nwords, nchunks));
    DSRG_LAUNCH(e, T_LAT_MISC, s,
                k_lattice_neighbors<D><<<gv, kThreads, 0, s>>>(L.hkeys, L.hval, L.vslot, L.vcount, L.rowbase,
                                                               L.nbr, L.nbr_stride, a.cap, L.capv, L.shared));
    DSRG_LAUNCH(e, T_LAT_MISC, s,
                k_lattice_cleanup<<<gv, kThreads, 0, s>>>(L.hkeys, L.hval, L.vslot, L.vcount, a.cap, L.capv));
    return DSRG_OK;
}

// Read-out for the tests (dsrg_engine_lattice_idle): the build-to-build state is all-empty hash slots, hval -1 and
// vkey kNoKey; counts what differs from it
__global__ void __launch_bounds__(kThreads)
k_lattice_idle(const uint64_t *hkeys, const int32_t *hval, long long nslots, const int32_t *vkey, long long nverts,
               unsigned long long *counts) {
    unsigned long long c[3] = {0, 0, 0};
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nslots; i += stride) {
        c[0] += hkeys[i] != kEmptyKey;
        c[1] += hval[i] != -1;
    }
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nverts; i += stride) c[2] += vkey[i] != kNoKey;
#pragma unroll
    for (int k = 0; k < 3; k++)
        if (c[k]) atomicAdd(counts + k, c[k]);
}

int lattice_idle(Engine *e, const Lattice &L, long long *counts) {
    DSRG_CUDA_TRY(cudaDeviceSynchronize());
    unsigned long long *d = nullptr;
    DSRG_CUDA_TRY(cudaMalloc(&d, 3 * sizeof(unsigned long long)));
    cudaError_t err = cudaMemset(d, 0, 3 * sizeof(unsigned long long));
    if (err == cudaSuccess) {  // a read-out, not part of any pass: not counted in the engine's launches
        k_lattice_idle<<<4 * e->sm_count, kThreads>>>(L.hkeys, L.hval, L.slots_alloc, L.vkey, L.verts_alloc, d);
        err = cudaGetLastError();
    }
    if (err == cudaSuccess) err = cudaMemcpy(counts, d, 3 * sizeof(long long), cudaMemcpyDeviceToHost);
    cudaFree(d);
    DSRG_CUDA_TRY(err);
    return DSRG_OK;
}

// Build the lattices of `B` images (or the single shared one), then their norm vectors.  `feat` ([B][5][N], the
// bilateral lattice only): the caller's features in place of the image's, with per-image range flags in `bad` [B].
int lattice_build(Engine *e, Lattice &L, int B, const uint8_t *image_dev, cudaStream_t s, const float *feat,
                  int *bad) {
    const int nb = L.shared ? 1 : B;
    int rc = (L.d == 2) ? build_impl<2>(e, L, nb, image_dev, nullptr, nullptr, s)
                        : build_impl<5>(e, L, nb, image_dev, feat, bad, s);
    if (rc) return rc;
    // norm pass on nb structures; value rows of the norm pass use the per-structure packing,
    // which for the shared lattice is simply image 0's rows [0, V+1).
    const int dp1 = L.d + 1;
    const long long rows_nb = L.shared ? (long long)L.capv + 1 : L.rows_cap;
    DSRG_CUDA_TRY(cudaMemsetAsync(e->nvA, 0, sizeof(float) * rows_nb, s));
    dim3 gp(cdiv(L.N, kThreads), nb);
    DSRG_LAUNCH(e, T_LAT_NORM, s, k_norm_splat<<<gp, kThreads, 0, s>>>(L.off, L.bary, L.rowbase, L.vkey, e->nvA, L.N, dp1, L.capv));
    float *src = e->nvA, *dst = e->nvB;
    for (int j = 0; j < dp1; j++) {
        DSRG_LAUNCH(e, T_LAT_NORM, s,
                    k_norm_blur<<<4 * e->sm_count, kThreads, 0, s>>>(src, dst, L.nbr + (size_t)j * L.nbr_stride,
                                                                      L.rowbase, nb));
        float *t = src;
        src = dst;
        dst = t;
    }
    const float alpha = 1.0f / (1 + powf(2, -L.d));  // permutohedral.cpp:510
    DSRG_LAUNCH(e, T_LAT_NORM, s, k_norm_slice<<<gp, kThreads, 0, s>>>(L.off, L.bary, L.rowbase, src, L.norm, L.N, dp1, alpha,
                                                                       L.vkey, L.vcount, L.capv));
    DSRG_CUDA_TRY(cudaGetLastError());
    // the tile-local views serve the fused kernel (up to DSRG_MAX_LABELS labels); the wide path only needs bary * norm
    return e->MP > DSRG_MAX_LABELS ? wide_weights(e, L, nb, s) : tiles_build(e, L, nb, s);
}

}  // namespace dsrg
