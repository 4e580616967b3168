// Tile-local lattice views (sm_90a).
//
// The permutohedral splat / slice of the reference touch, per pixel, d+1 lattice rows of 24
// floats each (CRF/src/permutohedral.cpp:545-553, :574-584).  Neighbouring pixels share most of
// their vertices, so a 32x8-pixel tile only touches a few dozen DISTINCT rows.  This kernel
// finds them once per lattice build: per tile the distinct rows with, for each, its segment of the
// transposed incidence (tl_hdr), per pixel the index into that list (tl_loc), and the incidence
// itself as a CSR grouped by local vertex whose entries are already in the form the mean-field
// kernel consumes (tl_pack: 16 bits, r << 8 | pixel's thread index, which locate both the pixel's Q row
// and its weight in the kernel's shared tables, common.cuh:kEntZero); the whole entry list of a tile is
// one 16-byte-aligned block for a bulk copy.  Local vertices are numbered
// by decreasing segment length.  Tiles with too many distinct rows keep their most-shared ones (hybrid tiles).
// The symmetric normalisation is folded into the weights: wn = bary * norm (pairwise.cpp:66,79).
// wn and tl_loc are written twice: planar per pixel (tl_loc, wn: the backward, the gradient passes) and per tile in
// [r][thread] blocks (tl_li, tl_w), which the forward tile kernels bulk-copy into their shared tables as they are.
#include "common.cuh"

namespace dsrg {

template <int DP1, int MAXA, int MAXLOC>
__global__ void __launch_bounds__(kTileThreads)
k_tile_build(const int32_t *off, const float *bary, const float *norm, int32_t *tl_nloc, uint8_t *tl_hy, int2 *tl_hdr,
             uint16_t *tl_pack, uint16_t *tl_loc, float *wn, float *tl_w, uint16_t *tl_li, int N, int W, int H,
             int tiles_x, int ntiles, int entcap, int tile_w, int2 *hy_list, int *hy_count) {
    constexpr int HS = kTileThreads * 8;  // >= kTileThreads*DP1 distinct rows in the worst case, power of two
    constexpr int HBITS = (HS == 1024) ? 10 : (HS == 2048) ? 11 : (HS == 4096) ? 12 : -1;
    static_assert(HBITS > 0, "hash size");
    static_assert(MAXLOC <= kTileThreads, "one scan element per thread");
    __shared__ int hkey[HS];
    __shared__ int hlv[HS];
    __shared__ int hcnt[HS];
    __shared__ int rows_s[MAXLOC];
    __shared__ int cnt[MAXLOC];
    __shared__ int ptr[MAXLOC + 1];
    __shared__ int wsum[kTileThreads / 32], wsum2[kTileThreads / 32];
    __shared__ int sfx[kTileThreads + 1];
    __shared__ int perm[MAXLOC];
    __shared__ int scnt[MAXLOC];
    __shared__ int hist[kTileThreads + 2];
    __shared__ int count, nsel, thr_s, extra_s, ticket, covered, total;

    const int tile = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int tx = tile % tiles_x, ty = tile / tiles_x;
    const int x = tx * tile_w + (tid & 31), y = ty * kTileH + (tid >> 5);
    const bool in = (tid & 31) < tile_w && x < W && y < H;
    const int pix = y * W + x;
    for (int i = tid; i < HS; i += kTileThreads) hkey[i] = -1;
    if (tid < MAXLOC) cnt[tid] = 0;
    if (tid == 0) {
        count = 0;
        nsel = 0;
        ticket = 0;
    }
    __syncthreads();

    int slot[DP1];
    float w[DP1];
    if (in) {
        const float nrm = norm[(size_t)b * N + pix];
#pragma unroll
        for (int r = 0; r < DP1; r++) {
            const size_t at = ((size_t)b * DP1 + r) * N + pix;
            const int row = off[at];
            w[r] = __fmul_rn(bary[at], nrm);
            wn[at] = w[r];
            unsigned s = ((unsigned)row * 2654435761u) >> (32 - HBITS);
            while (true) {
                int old = atomicCAS(&hkey[s], -1, row);
                if (old == -1) {
                    int lv = atomicAdd(&count, 1);
                    hlv[s] = lv;
                    if (lv < MAXLOC) rows_s[lv] = row;
                    break;
                }
                if (old == row) break;
                s = (s + 1) & (HS - 1);
            }
            slot[r] = (int)s;
        }
    }
    // this tile's blocks: slot tid of row r
    const size_t blk = ((size_t)b * ntiles + tile) * DP1 * kTileThreads + tid;
#pragma unroll
    for (int r = 0; r < DP1; r++) tl_w[blk + r * kTileThreads] = in ? w[r] : 0.0f;
    __syncthreads();
    tl_nloc += (size_t)b * ntiles;
    tl_hy += (size_t)b * ntiles;
    // A tile with more than MAXA distinct vertices (what k_mf_tile's shared memory holds) is an overflow tile.
    // Textured images produce them: their vertices are shared in colour space, not between neighbouring pixels.
    // If the MAXLOC most-touched vertices (two incidences or more each) cover a fair share of the tile's
    // incidences it becomes a HYBRID tile, run by k_mf_tile_hy: those vertices keep the tile-local CSR, the other
    // (pixel, vertex) incidences are marked kLocRemote in tl_loc and are sliced / splatted directly in global
    // memory.  Otherwise (uniform noise, the sigma/12 training lattices; always for the shared spatial lattice and
    // for small passes, hy_list == nullptr) nothing is kept: count -1, every incidence remote, k_mf_tile's direct path.
    const bool overflow = count > MAXA;
    bool hybrid = false;
    int lv[DP1];
    int nloc = count;
    if (!overflow) {
        if (in) {
#pragma unroll
            for (int r = 0; r < DP1; r++) {
                lv[r] = hlv[slot[r]];
                atomicAdd(&cnt[lv[r]], 1);
            }
        }
        __syncthreads();
    } else {
        hybrid = DP1 == 6 && hy_list != nullptr;
        if (hybrid) {
            for (int i = tid; i < HS; i += kTileThreads) hcnt[i] = 0;
            for (int i = tid; i < kTileThreads + 2; i += kTileThreads) hist[i] = 0;
            __syncthreads();
            if (in) {
#pragma unroll
                for (int r = 0; r < DP1; r++) atomicAdd(&hcnt[slot[r]], 1);  // incidences of the vertex inside the tile
            }
            __syncthreads();
            for (int i = tid; i < HS; i += kTileThreads)
                if (hkey[i] != -1) atomicAdd(&hist[hcnt[i]], 1);  // an incidence count is at most kTileThreads
            __syncthreads();
            // threshold = the smallest incidence count c >= 2 such that the vertices with count >= c fit into MAXLOC:
            // thread t stands for c = kTileThreads - t, so an inclusive scan over t yields the suffix sums over c
            {
                const int c = kTileThreads - tid;
                int nv = hist[c], ni = c * nv;  // vertices with exactly c incidences, and their incidences
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int a = __shfl_up_sync(0xffffffffu, nv, o), d = __shfl_up_sync(0xffffffffu, ni, o);
                    if ((tid & 31) >= o) {
                        nv += a;
                        ni += d;
                    }
                }
                if ((tid & 31) == 31) {
                    wsum[tid >> 5] = nv;
                    wsum2[tid >> 5] = ni;
                }
                __syncthreads();
                for (int k = 0; k < (tid >> 5); k++) {
                    nv += wsum[k];
                    ni += wsum2[k];
                }
                sfx[tid] = nv;
                __syncthreads();
                const bool ok = c >= 2 && nv <= MAXLOC;
                const bool next_ok = (c - 1 >= 2) && sfx[tid + 1] <= MAXLOC;  // tid + 1 <= kTileThreads - 2 here
                if (ok && !next_ok) {  // exactly one thread: every vertex with >= c incidences is local,
                    thr_s = c;
                    const int extra = (c - 1 >= 2) ? MAXLOC - nv : 0;  // and the first `extra` ones of the next bucket
                    extra_s = extra;
                    covered = ni + extra * (c - 1);
                }
                const int npix = __syncthreads_count(in);
                if (tid == 0) total = npix * DP1;
            }
            __syncthreads();
            hybrid = covered * 100 >= total * DSRG_HY_MIN_COVER;
        }
        if (!hybrid) {
            if (in) {
#pragma unroll
                for (int r = 0; r < DP1; r++) tl_loc[((size_t)b * DP1 + r) * N + pix] = (uint16_t)kLocRemote;
            }
#pragma unroll
            for (int r = 0; r < DP1; r++) tl_li[blk + r * kTileThreads] = (uint16_t)kLocRemote;
            if (tid == 0) {
                tl_nloc[tile] = -1;
                tl_hy[tile] = 0;
            }
            return;
        }
        const int thr = thr_s, extra = extra_s;
        for (int i = tid; i < HS; i += kTileThreads) {
            int l = -1;
            if (hkey[i] != -1) {
                const int c = hcnt[i];
                bool sel = c >= thr;
                if (!sel && c == thr - 1 && extra > 0) sel = atomicAdd(&ticket, 1) < extra;
                if (sel) {
                    l = atomicAdd(&nsel, 1);
                    rows_s[l] = hkey[i];
                    cnt[l] = c;
                }
            }
            hlv[i] = l;
        }
        __syncthreads();
        nloc = nsel;
        if (in) {
#pragma unroll
            for (int r = 0; r < DP1; r++) lv[r] = hlv[slot[r]];
        }
    }
    // order the local vertices by decreasing segment length so that the lanes of a warp of the
    // consumer (one lane per (vertex, label quad)) walk segments of similar length
    const int mycnt = tid < nloc ? cnt[tid] : 0;
    if (tid < nloc) {
        int rank = 0;
        for (int j = 0; j < nloc; j++) {
            const int cj = cnt[j];
            rank += (cj > mycnt) || (cj == mycnt && j < tid);
        }
        perm[tid] = rank;      // new index of local vertex `tid`
        scnt[rank] = mycnt;    // counts in the new order
    }
    __syncthreads();
    // exclusive scan of the reordered counts, each rounded up to an even number -> ptr: every segment then
    // starts on a 4-byte boundary and the consumer reads its entries two at a time (one LDS.32)
    {
        const int v = tid < nloc ? ((scnt[tid] + 1) & ~1) : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int n = __shfl_up_sync(0xffffffffu, incl, o);
            if ((tid & 31) >= o) incl += n;
        }
        if ((tid & 31) == 31) wsum[tid >> 5] = incl;
        __syncthreads();
        int base = 0;
        for (int k = 0; k < (tid >> 5); k++) base += wsum[k];
        if (tid < MAXLOC) {
            ptr[tid] = base + incl - v;
            cnt[tid] = 0;  // reused as the fill cursor (indexed by the NEW vertex index)
        }
    }
    __syncthreads();
    uint16_t *pack = tl_pack + ((size_t)b * ntiles + tile) * entcap;
    if (!in) {
#pragma unroll
        for (int r = 0; r < DP1; r++) tl_li[blk + r * kTileThreads] = (uint16_t)kLocRemote;
    } else {
#pragma unroll
        for (int r = 0; r < DP1; r++) {
            uint16_t *loc = tl_loc + ((size_t)b * DP1 + r) * N + pix;
            if (lv[r] < 0) {
                *loc = (uint16_t)kLocRemote;
                tl_li[blk + r * kTileThreads] = (uint16_t)kLocRemote;
                continue;
            }
            const int nv = perm[lv[r]];
            *loc = (uint16_t)nv;
            tl_li[blk + r * kTileThreads] = (uint16_t)nv;
            const int pos = ptr[nv] + atomicAdd(&cnt[nv], 1);
            pack[pos] = (uint16_t)((ent_r0(DP1) + r) << 8 | tid);  // its weight: slot tid of row r of the tile's tl_w block
        }
    }
    if (tid < nloc) {
        const int nv = perm[tid];
        tl_hdr[((size_t)b * ntiles + tile) * MAXLOC + nv] = make_int2(ptr[nv] | (mycnt << 16), rows_s[tid]);
        if (mycnt & 1) pack[ptr[nv] + mycnt] = (uint16_t)kEntZero;  // padding entry: pixel 0 with weight 0
    }
    if (tid == 0) {
        tl_nloc[tile] = nloc | (hybrid ? kTileHybrid : 0);
        tl_hy[tile] = hybrid ? 1 : 0;
        if (hybrid) hy_list[atomicAdd(hy_count, 1)] = make_int2(tile, b);  // k_mf_tile_hy's work list
    }
}

// A batch with only a few hybrid tiles (smooth images: the odd tile with 200 vertices) is better off without
// them: k_mf_tile_hy would run eleven nearly empty waves in line with the plain kernel.  Below `min_tiles` the
// listed tiles are handed back to k_mf_tile's direct path (count -1) and the list is emptied.
__global__ void __launch_bounds__(kThreads)
k_tile_demote(int2 *hy_list, int *hy_count, int32_t *tl_nloc, uint8_t *tl_hy, int ntiles, int min_tiles) {
    const int n = *hy_count;
    if (n >= min_tiles) return;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int2 t = hy_list[i];
        tl_nloc[(size_t)t.y * ntiles + t.x] = -1;
        tl_hy[(size_t)t.y * ntiles + t.x] = 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) *hy_count = 0;
}

int tiles_build(Engine *e, Lattice &L, int nb, cudaStream_t s) {
    dim3 g(e->ntiles, nb);
    const bool hy_on = L.d == 5 && hybrid_tiles_on(e, nb);
    if (L.d == 5) DSRG_CUDA_TRY(cudaMemsetAsync(e->hy_count, 0, sizeof(int), s));  // the list of hybrid tiles is rebuilt (or stays empty)
#define DSRG_TILE_BUILD(DP1, MAXA, MAXLOC)                                                                   \
    DSRG_LAUNCH(e, T_LAT_MISC, s,                                                                            \
                (k_tile_build<DP1, MAXA, MAXLOC><<<g, kTileThreads, 0, s>>>(L.off, L.bary, L.norm, L.tl_nloc, L.tl_hy, L.tl_hdr, \
                                                                  L.tl_pack, L.tl_loc, L.wn, L.tl_w, L.tl_li,  \
                                                                  L.N, e->W, e->H, e->tiles_x, e->ntiles,      \
                                                                  L.entcap, e->tile_w,                         \
                                                                  hy_on ? e->hy_list : nullptr, e->hy_count)))
    if (L.d == 2) DSRG_TILE_BUILD(3, kMaxLocSp, kMaxLocSp);
    else DSRG_TILE_BUILD(6, kMaxLocBi, kMaxLocHy);
    if (hy_on)
        DSRG_LAUNCH(e, T_LAT_MISC, s,
                    k_tile_demote<<<1, kThreads, 0, s>>>(e->hy_list, e->hy_count, L.tl_nloc, L.tl_hy, e->ntiles, DSRG_HY_MIN_TILES * e->sm_count));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

}  // namespace dsrg
