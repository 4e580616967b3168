// Mean-field inference of the fully connected CRF (sm_90a).
//
// Replaces DenseCRF::inference (CRF/src/densecrf.cpp:115-131) with its per-iteration calls
// PairwisePotential::apply -> DenseKernel::filter -> Permutohedral::sseCompute ->
// PottsCompatibility::apply (CRF/src/pairwise.cpp:173-178, :63-80; permutohedral.cpp:529-589;
// labelcompatibility.cpp:46-48) and expAndNormalize (densecrf.cpp:98-106), for the whole batch.
//
// State is planar: U, Q are [B][M][N] float32 (one coalesced load per label per thread);
// lattice value rows are [rows][MP] float32 with MP = M rounded up to a multiple of 4
// (the reference pads 21 -> 24 the same way, permutohedral.cpp:531).
#include "common.cuh"

namespace dsrg {

// ---------------------------------------------------------------------------------------------
// init: unary (any layout) -> U planar; Q = softmax(U)   (densecrf.cpp:120 with energy = -unary)
// ---------------------------------------------------------------------------------------------
template <int MP>
__global__ void __launch_bounds__(kThreads)
k_mf_init(const float *unary, float *unary_rw, int layout, int clamp, float *U, float *Q, int M,
          int N) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    float u[MP];
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < MP; k++) {
        if (k < M) {
            size_t at = (layout == DSRG_LAYOUT_NCHW) ? ((size_t)b * M + k) * N + i
                                                     : ((size_t)b * N + i) * M + k;
            float v = unary[at];
            if (clamp && v < kMinProb) {  // probs[probs < min_prob] = min_prob, pylayers.py:312
                v = kMinProb;
                unary_rw[at] = v;
            }
            u[k] = v;
            mx = fmaxf(mx, v);
        }
    }
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < MP; k++)
        if (k < M) {
            U[((size_t)b * M + k) * N + i] = u[k];
            u[k] = expf(u[k] - mx);
            s += u[k];
        }
    if (Q) {
#pragma unroll
        for (int k = 0; k < MP; k++)
            if (k < M) Q[((size_t)b * M + k) * N + i] = u[k] / s;
    }
}

// ---------------------------------------------------------------------------------------------
// The fused per-iteration kernel: one CTA per 32x8-pixel tile, one thread per pixel.
//
//   slice  : out_i = sum_r (bary_r alpha) values[row_r]            (permutohedral.cpp:574-584)
//   update : t = U + w2 norm_sp out_sp + w1 norm_bi out_bi ; Q = softmax(t)
//            (pairwise.cpp:79, labelcompatibility.cpp:46-48, densecrf.cpp:123-128, :98-106)
//   splat  : values'[row_r] += bary_r (Q_i norm_i)                  (pairwise.cpp:66, permutohedral.cpp:545-553)
//
// Fusing the slice of iteration t with the splat of iteration t+1 means Q never goes to HBM
// between iterations: per iteration the kernel streams U once (4*M*N bytes per image) plus the
// tile-local lattice view.  The rows a tile touches are staged in shared memory once (slice), the
// new marginals are parked in shared memory, and the splat walks the tile's CSR (entries grouped
// by local vertex) so that each distinct vertex receives ONE vectorised global reduction
// (REDG.ADD.F32x4) per tile instead of one scalar atomic per pixel, vertex and label.
// norm is folded into the weights (wn = bary*norm, built in tiles.cu).
// Tiles that touch more distinct vertices than fit take the direct global path (count -1: uniform noise, sigma/12
// lattices) or, when a few vertices carry most of their incidences (textured images), are hybrid tiles and belong to
// k_mf_tile_hy below (tiles.cu decides).
// ---------------------------------------------------------------------------------------------
struct TileLat {
    // direct view (overflow tiles, remote incidences of hybrid tiles)
    const int32_t *off;      // [nimg][dp1][N] local row (1-based)
    const int32_t *rowbase;  // [B+1]
    // tile-local view (tiles.cu)
    const int32_t *tl_nloc;
    const uint8_t *tl_hy;    // [nimg][ntiles] 1: hybrid tile (bilateral view only)
    const int2 *tl_hdr;
    const uint16_t *tl_pack;
    const uint16_t *tl_loc;
    const float *wn;         // [nimg][dp1][N]
    const float *val_in;     // blurred values of the previous splat (slice source)
    float *val_out;          // zeroed values (splat target)
    int entcap;
    int shared;
};

enum { MODE_FIRST = 0, MODE_MID = 1, MODE_LAST = 2 };

// exp(x) for x <= 0 via ex2.approx with the rounding error of x*log2(e) folded back in
// (relative error ~2^-22, independent of |x|)
__device__ __forceinline__ float exp_neg(float x) {
    const float kL2E = 1.4426950408889634f, kL2E_lo = 1.9259630e-8f, kLn2 = 0.6931471805599453f;
    const float t = x * kL2E;
    float r = fmaf(x, kL2E, -t);
    r = fmaf(x, kL2E_lo, r);
    float e;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
    return fmaf(e, r * kLn2, e);
}

// ---- mbarrier + 1-D bulk copy (TMA engine, SASS UBLKCP) ------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// bounded wait: a protocol bug must surface as a launch failure, never as a hung GPU
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    for (uint32_t spin = 0; !mbar_try_wait(bar, parity); ++spin)
        if (spin > (1u << 24)) __trap();
}
// global -> shared, size and both addresses multiples of 16 bytes; completion is signalled on `bar`
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

template <int MP>
struct TileRow {
    static constexpr int CH = MP / 4;
    static constexpr int CHP = CH + DSRG_ROW_PAD;  // float4 per staged row (padded)
};

// A tile's staging area: its local vertices' value rows (later its Q rows), its CSR entry blocks and the mbarrier
// the bulk copies complete on; TileSmem adds the weight table the entries index.
template <int MP, int MAXBI = kMaxLocBi>
struct TileStage {
    static constexpr int CH = MP / 4;
    static constexpr int CHP = TileRow<MP>::CHP;
    static constexpr int kRows = kMaxLocSp + MAXBI;
    static constexpr int kBufF4 = (kRows * CHP > kTileThreads * CHP) ? kRows * CHP : kTileThreads * CHP;  // staged rows / Q alias
    // segments padded to even, each block a whole number of 16-byte units
    static constexpr int kEntSp = (kTileThreads * 3 + kMaxLocSp + 7) & ~7, kEntBi = (kTileThreads * 6 + MAXBI + 7) & ~7;
    float4 buf[kBufF4];
    uint16_t ent[kEntSp + kEntBi];  // CSR entries (r << 8 | thread, common.cuh:kEntZero)
    uint64_t bar;
};

template <int MP, int MAXBI = kMaxLocBi>
struct TileSmem {
    TileStage<MP, MAXBI> st;
    float wtab[kEntZero + 4];  // [r][thread] weights of the tile being splatted, then the zero slot
};

// the size of a lattice's CSR entry block as bulk-copied, from the header of its last segment
__device__ __forceinline__ uint32_t ent_block_bytes(int2 last) {
    return ((uint32_t)((last.x & 0xffff) + (((last.x >> 16) + 1) & ~1)) * 2u + 15u) & ~15u;
}

// the current tile's weights into the table its CSR entries index; the CTA's thread t is the tile's pixel t
__device__ __forceinline__ void tile_put_weights(float *wtab, const float *w_sp, const float *w_bi) {
#pragma unroll
    for (int r = 0; r < 3; r++) wtab[(ent_r0(3) + r) * kTileThreads + threadIdx.x] = w_sp[r];
#pragma unroll
    for (int r = 0; r < 6; r++) wtab[(ent_r0(6) + r) * kTileThreads + threadIdx.x] = w_bi[r];
}

// slice one lattice from the staged rows (shared memory): t += coef * sum_r wn_r * row_r
// tail1: M = MP - 3 (e.g. 21 labels in 24 lanes): the last chunk holds ONE real channel, so a 32-bit load
// (one shared-memory wavefront per warp) replaces the 128-bit one (four)
template <int MP, int DP1>
__device__ __forceinline__ void tile_slice_smem(const float4 *vs, const uint16_t *loc, size_t stride,
                                                const float *w, float coef, float *t, bool tail1) {
    constexpr int CH = MP / 4, CHP = TileRow<MP>::CHP;
#pragma unroll
    for (int r = 0; r < DP1; r++) {
        const float4 *row = vs + (int)__ldg(loc + r * stride) * CHP;
        const float wr = coef * w[r];
#pragma unroll
        for (int c = 0; c < CH - 1; c++) {
            const float4 v = row[c];
            t[4 * c + 0] = fmaf(wr, v.x, t[4 * c + 0]);
            t[4 * c + 1] = fmaf(wr, v.y, t[4 * c + 1]);
            t[4 * c + 2] = fmaf(wr, v.z, t[4 * c + 2]);
            t[4 * c + 3] = fmaf(wr, v.w, t[4 * c + 3]);
        }
        constexpr int c = CH - 1;
        if (tail1) {
            const float v = reinterpret_cast<const float *>(row + c)[0];
            t[4 * c + 0] = fmaf(wr, v, t[4 * c + 0]);
        } else {
            const float4 v = row[c];
            t[4 * c + 0] = fmaf(wr, v.x, t[4 * c + 0]);
            t[4 * c + 1] = fmaf(wr, v.y, t[4 * c + 1]);
            t[4 * c + 2] = fmaf(wr, v.z, t[4 * c + 2]);
            t[4 * c + 3] = fmaf(wr, v.w, t[4 * c + 3]);
        }
    }
}

// fallback: slice straight from the global value rows
template <int MP, int DP1>
__device__ __forceinline__ void tile_slice_global(const float4 *vin, const int32_t *off, size_t stride,
                                                  int base, const float *w, float coef, float *t) {
    constexpr int CH = MP / 4;
#pragma unroll
    for (int r = 0; r < DP1; r++) {
        const float4 *row = vin + (size_t)(base + off[r * stride]) * CH;
        const float wr = coef * w[r];
#pragma unroll
        for (int c = 0; c < CH; c++) {
            const float4 v = row[c];
            t[4 * c + 0] = fmaf(wr, v.x, t[4 * c + 0]);
            t[4 * c + 1] = fmaf(wr, v.y, t[4 * c + 1]);
            t[4 * c + 2] = fmaf(wr, v.z, t[4 * c + 2]);
            t[4 * c + 3] = fmaf(wr, v.w, t[4 * c + 3]);
        }
    }
}

// hybrid tiles (tiles.cu): an incidence whose vertex is in the tile-local list is sliced from the staged rows, the
// others (tl_loc == kLocRemote) straight from the global value rows; returns the mask of the remote ones
template <int MP, int DP1>
__device__ __forceinline__ unsigned tile_slice_mixed(const float4 *vs, const uint16_t *loc, const float4 *vin,
                                                     const int32_t *off, size_t stride, int base, const float *w,
                                                     float coef, float *t) {
    constexpr int CH = MP / 4, CHP = TileRow<MP>::CHP;
    unsigned remote = 0;  // bit r: incidence r of this pixel goes direct
#pragma unroll
    for (int r = 0; r < DP1; r++) {
        const int l = (int)__ldg(loc + r * stride);
        const float wr = coef * w[r];
        if (l != kLocRemote) {
            const float4 *row = vs + l * CHP;
#pragma unroll
            for (int c = 0; c < CH; c++) {
                const float4 v = row[c];
                t[4 * c + 0] = fmaf(wr, v.x, t[4 * c + 0]);
                t[4 * c + 1] = fmaf(wr, v.y, t[4 * c + 1]);
                t[4 * c + 2] = fmaf(wr, v.z, t[4 * c + 2]);
                t[4 * c + 3] = fmaf(wr, v.w, t[4 * c + 3]);
            }
        } else {
            remote |= 1u << r;
            const float4 *row = vin + (size_t)(base + __ldg(off + r * stride)) * CH;
#pragma unroll
            for (int c = 0; c < CH; c++) {
                const float4 v = __ldg(row + c);
                t[4 * c + 0] = fmaf(wr, v.x, t[4 * c + 0]);
                t[4 * c + 1] = fmaf(wr, v.y, t[4 * c + 1]);
                t[4 * c + 2] = fmaf(wr, v.z, t[4 * c + 2]);
                t[4 * c + 3] = fmaf(wr, v.w, t[4 * c + 3]);
            }
        }
    }
    return remote;
}

// which incidences of this pixel are remote (first iteration: nothing is sliced)
template <int DP1>
__device__ __forceinline__ unsigned tile_remote_mask(const uint16_t *loc, size_t stride) {
    unsigned remote = 0;
#pragma unroll
    for (int r = 0; r < DP1; r++)
        if ((int)__ldg(loc + r * stride) == kLocRemote) remote |= 1u << r;
    return remote;
}

// CSR splat of both lattices: one thread per (local vertex, label quad) walks the vertex's segment
// serially and issues ONE vector reduction; vertices are ordered by segment length (tiles.cu), so the
// lanes of a warp run similar trip counts, and no cross-lane reduction is needed.
// An entry e names the pixel's Q row (e & 255) and its weight wtab[e].
template <int MP>
__device__ __forceinline__ void tile_splat_csr(float4 *vout_sp, float4 *vout_bi, int n_sp, int n_bi,
                                               const int2 *hdr_sp, const int2 *hdr_bi, int base_sp, int base_bi,
                                               const uint16_t *ent_sp, const uint16_t *ent_bi, const float4 *qs,
                                               const float *wtab) {
    constexpr int CH = MP / 4, CHP = TileRow<MP>::CHP;
    // 8 lanes per vertex (CH of them active): every quarter-warp of an LDS.128 then reads ONE pixel
    // row (contiguous 96 B), which is bank-conflict free (packing CH lanes is not)
    constexpr int LPV = 8;
    constexpr int kPairUnroll = kSplatUnroll / 2 > 0 ? kSplatUnroll / 2 : 1;
    static_assert(CH <= LPV, "lane mapping");
    const int pairs_sp = n_sp * LPV, pairs = (n_sp + n_bi) * LPV;
    const int cq = threadIdx.x & (LPV - 1);  // 256 % LPV == 0: a thread keeps its label quad
    if (cq >= CH) return;
    // the headers live in global memory (L1/L2-resident): the next task's header is fetched while the
    // current segment is walked
    auto hdr_of = [&](int p) {
        const bool s = p < pairs_sp;
        return __ldg((s ? hdr_sp : hdr_bi) + (s ? p : p - pairs_sp) / LPV);
    };
    int2 hn = threadIdx.x < pairs ? hdr_of(threadIdx.x) : make_int2(0, 0);
    for (int p = threadIdx.x; p < pairs; p += kTileThreads) {
        const bool is_sp = p < pairs_sp;
        const int2 h = hn;  // (first entry | count << 16, local row id)
        if (p + kTileThreads < pairs) hn = hdr_of(p + kTileThreads);
        // segments start on even entries and are padded to an even count (weight-0 entry): two per load
        const uint32_t *ep = reinterpret_cast<const uint32_t *>((is_sp ? ent_sp : ent_bi) + (h.x & 0xffff));
        const int n2 = ((h.x >> 16) + 1) >> 1;
        const float4 *qb = qs + cq;
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll kPairUnroll
        for (int it = 0; it < n2; ++it) {
            const uint32_t en = ep[it];
            const uint32_t e0 = en & 0xffffu, e1 = en >> 16;
            const float w0 = wtab[e0], w1 = wtab[e1];
            const float4 q0 = qb[(e0 & 255u) * CHP];
            const float4 q1 = qb[(e1 & 255u) * CHP];
            a.x = fmaf(w0, q0.x, a.x);
            a.y = fmaf(w0, q0.y, a.y);
            a.z = fmaf(w0, q0.z, a.z);
            a.w = fmaf(w0, q0.w, a.w);
            a.x = fmaf(w1, q1.x, a.x);
            a.y = fmaf(w1, q1.y, a.y);
            a.z = fmaf(w1, q1.z, a.z);
            a.w = fmaf(w1, q1.w, a.w);
        }
        atomicAdd((is_sp ? vout_sp : vout_bi) + (size_t)((is_sp ? base_sp : base_bi) + h.y) * CH + cq, a);
    }
}

// direct splat of one pixel (fallback tiles): d+1 rows x MP/4 vector reductions
template <int MP, int DP1>
__device__ __forceinline__ void tile_splat_direct(float4 *vout, const int32_t *off, size_t stride,
                                                  int base, const float *w, const float *q) {
    constexpr int CH = MP / 4;
#pragma unroll
    for (int r = 0; r < DP1; r++) {
        float4 *row = vout + (size_t)(base + off[r * stride]) * CH;
#pragma unroll
        for (int c = 0; c < CH; c++)
            atomicAdd(row + c, make_float4(w[r] * q[4 * c], w[r] * q[4 * c + 1], w[r] * q[4 * c + 2],
                                           w[r] * q[4 * c + 3]));
    }
}

// direct splat of one pixel's remote incidences (hybrid tiles): MP/4 vector reductions per such row
template <int MP, int DP1>
__device__ __forceinline__ void tile_splat_remote(float4 *vout, unsigned remote, const int32_t *off, size_t stride,
                                                  int base, const float *w, const float *q) {
    constexpr int CH = MP / 4;
#pragma unroll
    for (int r = 0; r < DP1; r++) {
        if (!(remote >> r & 1u)) continue;
        float4 *row = vout + (size_t)(base + __ldg(off + r * stride)) * CH;
#pragma unroll
        for (int c = 0; c < CH; c++)
            atomicAdd(row + c, make_float4(w[r] * q[4 * c], w[r] * q[4 * c + 1], w[r] * q[4 * c + 2],
                                           w[r] * q[4 * c + 3]));
    }
}

// ---- the per-tile steps both tile kernels share ----
// The tile coordinates and the bulk-copy staging are still written out in each kernel: moved into a shared helper,
// either one changed the SASS of some k_mf_tile / k_mf_tile_hy instantiations (register choice, loop offsets).
//
// Park the pixel's Q row in the staging buffer (once every thread is done reading the staged rows) and its weights
// in wtab, for the CSR splat; returns the Q rows
template <int MP, int MAXBI>
__device__ __forceinline__ const float4 *tile_park(TileSmem<MP, MAXBI> &smt, const float *t, const float *w_sp,
                                                   const float *w_bi) {
    constexpr int CH = MP / 4, CHP = TileStage<MP, MAXBI>::CHP;
    const int tid = threadIdx.x;
    __syncthreads();
    float4 *qs = smt.st.buf;
#pragma unroll
    for (int c = 0; c < CH; c++) qs[tid * CHP + c] = make_float4(t[4 * c], t[4 * c + 1], t[4 * c + 2], t[4 * c + 3]);
    tile_put_weights(smt.wtab, w_sp, w_bi);
    __syncthreads();
    return qs;
}

// Q = softmax(t) in place (expAndNormalize, densecrf.cpp:98-106); the last iteration stores it to Qout
template <int MP, int MODE>
__device__ __forceinline__ void tile_update(float *t, int M, int N, float *__restrict__ Qout, int b, int pix, bool in) {
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < MP; k++)
        if (k < M) mx = fmaxf(mx, t[k]);
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < MP; k++) {
        t[k] = (k < M) ? exp_neg(t[k] - mx) : 0.0f;
        s += t[k];
    }
    const float inv = __frcp_rn(s);
#pragma unroll
    for (int k = 0; k < MP; k++) t[k] *= inv;
    if (MODE == MODE_LAST) {
        if (in) {
            float *Qb = Qout + (size_t)b * M * N + pix;
#pragma unroll
            for (int k = 0; k < MP; k++) {
                if (k < M) *Qb = t[k];
                Qb += N;
            }
        }
    }
}

// The pixel's unaries into t and its folded weights into w_sp / w_bi (zeros outside the image).  U is either the
// engine's planar copy or, for NCHW callers, the caller's buffer itself; the reference's in-place clamp
// (pylayers.py:312) is then applied on the fly and written back once, by the first iteration.
template <int MP, int MODE>
__device__ __forceinline__ void tile_load_pixel(const float *U, float *U_rw, int clamp, int M, int N, int b, int pix,
                                                bool in, const float *wn_sp, const float *wn_bi, float *t,
                                                float *w_sp, float *w_bi) {
    {
        const size_t ub = (size_t)b * M * N + pix;
        const float *Ub = U + ub;
#pragma unroll
        for (int k = 0; k < MP; k++) {
            float v = 0.0f;
            if (in && k < M) v = (MODE == MODE_FIRST) ? *Ub : __ldg(Ub);  // read-only path once nothing writes U
            if (MODE == MODE_FIRST) {  // later iterations read the values this one wrote back
                if (clamp && in && k < M && v < kMinProb) {
                    v = kMinProb;
                    U_rw[ub + (size_t)k * N] = v;
                }
            }
            t[k] = v;
            Ub += N;
        }
    }
    {
        const float *p = wn_sp;
#pragma unroll
        for (int r = 0; r < 3; r++, p += N) w_sp[r] = in ? __ldg(p) : 0.0f;
        p = wn_bi;
#pragma unroll
        for (int r = 0; r < 6; r++, p += N) w_bi[r] = in ? __ldg(p) : 0.0f;
    }
}

template <int MP, int MODE>
__global__ void __launch_bounds__(kTileThreads, DSRG_TILE_CTAS)
k_mf_tile(const float *U, float *U_rw, int clamp, float *__restrict__ Qout, TileLat sp, TileLat bi, float c_sp,
          float c_bi, int M, int N, int W, int H, int tiles_x, int ntiles, int tile_w) {
    constexpr int kRowBytes = MP * 4;
    using SM = TileSmem<MP>;
    using ST = TileStage<MP>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    SM &smt = *reinterpret_cast<SM *>(smem_raw);
    ST &sm = smt.st;
    // A hybrid tile is k_mf_tile_hy's.  The test reads a byte map of its own and stands before anything else: the
    // same test on the tile's vertex count, wherever it was placed, made ptxas allocate this kernel's 64 registers
    // differently (more spill traffic in the splat loop, also on images that have no such tile at all).
    if (bi.tl_hy[(size_t)blockIdx.y * ntiles + blockIdx.x]) return;
    const int tile = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int tx = tile % tiles_x, ty = tile / tiles_x;
    const int x = tx * tile_w + (tid & 31), y = ty * kTileH + (tid >> 5);
    const bool in = (tid & 31) < tile_w && x < W && y < H;
    const int pix = in ? y * W + x : 0;
    const int sb_sp = sp.shared ? 0 : b, sb_bi = bi.shared ? 0 : b;
    const size_t ti_sp = (size_t)sb_sp * ntiles + tile, ti_bi = (size_t)sb_bi * ntiles + tile;
    const int nl_sp = sp.tl_nloc[ti_sp], nl_bi = bi.tl_nloc[ti_bi];
    const bool fb_sp = nl_sp < 0, fb_bi = nl_bi < 0;
    const int n_sp = fb_sp ? 0 : nl_sp, n_bi = fb_bi ? 0 : nl_bi;
    const int base_sp = sp.rowbase[b], base_bi = bi.rowbase[b];
    constexpr int CHP = ST::CHP;
    float4 *vs_sp = sm.buf, *vs_bi = sm.buf + kMaxLocSp * CHP;
    const int2 *hdr_sp = sp.tl_hdr + ti_sp * kMaxLocSp, *hdr_bi = bi.tl_hdr + ti_bi * kMaxLocHy;  // global, L1/L2-resident
    uint16_t *ent_sp = sm.ent, *ent_bi = sm.ent + ST::kEntSp;
    const size_t strideN = (size_t)N;
    const size_t px_sp = (size_t)sb_sp * 3 * N + pix, px_bi = (size_t)sb_bi * 6 * N + pix;

    // ---- asynchronous staging: every local vertex's value row (96 B) and the two CSR entry blocks
    // are pulled into shared memory by the bulk-copy engine while the threads load their per-pixel data
    const int n_copies = (MODE != MODE_FIRST ? n_sp + n_bi : 0) + (MODE != MODE_LAST ? (n_sp > 0) + (n_bi > 0) : 0);
    if (tid == 0) {
        mbar_init(&sm.bar, n_copies > 0 ? n_copies : 1);
        smt.wtab[kEntZero] = 0.0f;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    for (int i = tid; i < n_sp + n_bi; i += kTileThreads) {  // up to kMaxLocSp + kMaxLocBi local vertices
        const bool is_sp = i < n_sp;
        const int lv = is_sp ? i : i - n_sp;
        const int2 h = __ldg((is_sp ? hdr_sp : hdr_bi) + lv);
        const int row = (is_sp ? base_sp : base_bi) + h.y;
        if (MODE != MODE_FIRST) {
            mbar_arrive_expect_tx(&sm.bar, kRowBytes);
            bulk_g2s((is_sp ? vs_sp : vs_bi) + lv * CHP, (is_sp ? sp.val_in : bi.val_in) + (size_t)row * MP,
                     kRowBytes, &sm.bar);
        }
        if (MODE != MODE_LAST && lv == (is_sp ? n_sp : n_bi) - 1) {  // the last segment tells the block's length
            const uint32_t bytes = ent_block_bytes(h);
            mbar_arrive_expect_tx(&sm.bar, bytes);
            bulk_g2s(is_sp ? ent_sp : ent_bi,
                     is_sp ? sp.tl_pack + ti_sp * sp.entcap : bi.tl_pack + ti_bi * bi.entcap, bytes, &sm.bar);
        }
    }
    if (n_copies == 0 && tid == 0) mbar_arrive_expect_tx(&sm.bar, 0);

    // ---- per-pixel data (thread = pixel) ----
    float t[MP], w_sp[3], w_bi[6];
    tile_load_pixel<MP, MODE>(U, U_rw, clamp, M, N, b, pix, in, sp.wn + px_sp, bi.wn + px_bi, t, w_sp, w_bi);
    mbar_wait(&sm.bar, 0);

    // ---- slice + update ----
#ifdef DSRG_NO_TAIL1
    const bool tail1 = false;
#else
    const bool tail1 = (M == MP - 3);
#endif
    if (MODE != MODE_FIRST && in) {
        if (!fb_sp)
            tile_slice_smem<MP, 3>(vs_sp, sp.tl_loc + px_sp, strideN, w_sp, c_sp, t, tail1);
        else
            tile_slice_global<MP, 3>(reinterpret_cast<const float4 *>(sp.val_in), sp.off + px_sp, strideN,
                                     base_sp, w_sp, c_sp, t);
        if (!fb_bi)
            tile_slice_smem<MP, 6>(vs_bi, bi.tl_loc + px_bi, strideN, w_bi, c_bi, t, tail1);
        else
            tile_slice_global<MP, 6>(reinterpret_cast<const float4 *>(bi.val_in), bi.off + px_bi, strideN,
                                     base_bi, w_bi, c_bi, t);
    }
    tile_update<MP, MODE>(t, M, N, Qout, b, pix, in);
    if (MODE == MODE_LAST) return;
    const float4 *qs = tile_park(smt, t, w_sp, w_bi);
    // ---- splat ----
    float4 *vout_sp = reinterpret_cast<float4 *>(sp.val_out), *vout_bi = reinterpret_cast<float4 *>(bi.val_out);
    if (fb_sp && in) tile_splat_direct<MP, 3>(vout_sp, sp.off + px_sp, strideN, base_sp, w_sp, t);
    if (fb_bi && in) tile_splat_direct<MP, 6>(vout_bi, bi.off + px_bi, strideN, base_bi, w_bi, t);
    tile_splat_csr<MP>(vout_sp, vout_bi, n_sp, n_bi, hdr_sp, hdr_bi, base_sp, base_bi, ent_sp, ent_bi, qs, smt.wtab);
}

// Hybrid tiles (tiles.cu: more distinct vertices than the shared-memory path of k_mf_tile holds -- textured images,
// whose vertices are shared in colour space rather than between neighbouring pixels).  A persistent grid walks the
// list of such tiles: the kMaxLocHy most-touched vertices of a tile go through shared memory exactly like in
// k_mf_tile (bulk-copied rows, CSR splat), the remaining incidences are sliced from and reduced into global
// memory straight from the registers.  Its own register / shared-memory budget (DSRG_HY_CTAS CTAs per SM) keeps
// this code out of k_mf_tile's 64-register allocation.
template <int MP, int MODE>
__global__ void __launch_bounds__(kTileThreads, DSRG_HY_CTAS)
k_mf_tile_hy(const float *U, float *U_rw, int clamp, float *__restrict__ Qout, TileLat sp, TileLat bi, float c_sp,
             float c_bi, int M, int N, int W, int H, int tiles_x, int ntiles, int tile_w, const int2 *hy_list,
             const int *hy_count) {
    constexpr int kRowBytes = MP * 4;
    using ST = TileStage<MP, kMaxLocHy>;
    constexpr int CHP = ST::CHP;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    TileSmem<MP, kMaxLocHy> &smt = *reinterpret_cast<TileSmem<MP, kMaxLocHy> *>(smem_raw);
    ST &sm = smt.st;
    const int tid = threadIdx.x;
    const int nhy = *hy_count;
    const size_t strideN = (size_t)N;
    float4 *vs_sp = sm.buf, *vs_bi = sm.buf + kMaxLocSp * CHP;
    uint16_t *ent_sp = sm.ent, *ent_bi = sm.ent + ST::kEntSp;
    if (tid == 0) smt.wtab[kEntZero] = 0.0f;  // visible after the first tile's barriers
    float4 *vout_sp = reinterpret_cast<float4 *>(sp.val_out), *vout_bi = reinterpret_cast<float4 *>(bi.val_out);
    for (int item = blockIdx.x; item < nhy; item += gridDim.x) {
        const int2 bt = hy_list[item];
        const int tile = bt.x, b = bt.y;
        const int tx = tile % tiles_x, ty = tile / tiles_x;
        const int x = tx * tile_w + (tid & 31), y = ty * kTileH + (tid >> 5);
        const bool in = (tid & 31) < tile_w && x < W && y < H;
        const int pix = in ? y * W + x : 0;
        const int sb_sp = sp.shared ? 0 : b, sb_bi = bi.shared ? 0 : b;
        const size_t ti_sp = (size_t)sb_sp * ntiles + tile, ti_bi = (size_t)sb_bi * ntiles + tile;
        const int nl_sp = sp.tl_nloc[ti_sp], nl_bi = bi.tl_nloc[ti_bi];
        // a negative count is an overflow tile that kept no local list: all its incidences are remote
        const bool hy_sp = nl_sp < 0, hy_bi = true;
        const int n_sp = nl_sp < 0 ? 0 : nl_sp, n_bi = nl_bi & 0xffff;
        const int base_sp = sp.rowbase[b], base_bi = bi.rowbase[b];
        const int2 *hdr_sp = sp.tl_hdr + ti_sp * kMaxLocSp, *hdr_bi = bi.tl_hdr + ti_bi * kMaxLocHy;
        const size_t px_sp = (size_t)sb_sp * 3 * N + pix, px_bi = (size_t)sb_bi * 6 * N + pix;

        // ---- asynchronous staging of the local vertices' rows and the CSR entry blocks (as in k_mf_tile) ----
        const int n_copies = (MODE != MODE_FIRST ? n_sp + n_bi : 0) + (MODE != MODE_LAST ? (n_sp > 0) + (n_bi > 0) : 0);
        if (tid == 0) {
            mbar_init(&sm.bar, n_copies > 0 ? n_copies : 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        // the previous tile of this CTA wrote its Q rows into the same shared memory through the generic proxy: order
        // those writes before the bulk copies (async proxy) of this tile
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        for (int i = tid; i < n_sp + n_bi; i += kTileThreads) {
            const bool is_sp = i < n_sp;
            const int lv = is_sp ? i : i - n_sp;
            const int2 h = __ldg((is_sp ? hdr_sp : hdr_bi) + lv);
            const int row = (is_sp ? base_sp : base_bi) + h.y;
            if (MODE != MODE_FIRST) {
                mbar_arrive_expect_tx(&sm.bar, kRowBytes);
                bulk_g2s((is_sp ? vs_sp : vs_bi) + lv * CHP, (is_sp ? sp.val_in : bi.val_in) + (size_t)row * MP,
                         kRowBytes, &sm.bar);
            }
            if (MODE != MODE_LAST && lv == (is_sp ? n_sp : n_bi) - 1) {  // the last segment tells the block's length
                const uint32_t bytes = ent_block_bytes(h);
                mbar_arrive_expect_tx(&sm.bar, bytes);
                bulk_g2s(is_sp ? ent_sp : ent_bi,
                         is_sp ? sp.tl_pack + ti_sp * sp.entcap : bi.tl_pack + ti_bi * bi.entcap, bytes, &sm.bar);
            }
        }
        if (n_copies == 0 && tid == 0) mbar_arrive_expect_tx(&sm.bar, 0);

        // ---- per-pixel data ----
        float t[MP], w_sp[3], w_bi[6];
        tile_load_pixel<MP, MODE>(U, U_rw, clamp, M, N, b, pix, in, sp.wn + px_sp, bi.wn + px_bi, t, w_sp, w_bi);
        mbar_wait(&sm.bar, 0);

        // ---- slice + update ----
        unsigned rm_sp = 0, rm_bi = 0;  // this pixel's incidences that go direct
        if (in) {
            if (MODE != MODE_FIRST) {
                rm_sp = tile_slice_mixed<MP, 3>(vs_sp, sp.tl_loc + px_sp, reinterpret_cast<const float4 *>(sp.val_in),
                                                sp.off + px_sp, strideN, base_sp, w_sp, c_sp, t);
                rm_bi = tile_slice_mixed<MP, 6>(vs_bi, bi.tl_loc + px_bi, reinterpret_cast<const float4 *>(bi.val_in),
                                                bi.off + px_bi, strideN, base_bi, w_bi, c_bi, t);
            } else {
                if (hy_sp) rm_sp = tile_remote_mask<3>(sp.tl_loc + px_sp, strideN);
                if (hy_bi) rm_bi = tile_remote_mask<6>(bi.tl_loc + px_bi, strideN);
            }
        }
        tile_update<MP, MODE>(t, M, N, Qout, b, pix, in);
        if (MODE != MODE_LAST) {
            // ---- splat: remote incidences straight from the registers, the local vertices through the CSR ----
            if (rm_sp) tile_splat_remote<MP, 3>(vout_sp, rm_sp, sp.off + px_sp, strideN, base_sp, w_sp, t);
            if (rm_bi) tile_splat_remote<MP, 6>(vout_bi, rm_bi, bi.off + px_bi, strideN, base_bi, w_bi, t);
            const float4 *qs = tile_park(smt, t, w_sp, w_bi);
            tile_splat_csr<MP>(vout_sp, vout_bi, n_sp, n_bi, hdr_sp, hdr_bi, base_sp, base_bi, ent_sp, ent_bi, qs,
                               smt.wtab);
        }
        __syncthreads();  // the tile is done with the shared buffers and the barrier
        if (tid == 0) asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(smem_u32(&sm.bar)) : "memory");
    }
}

// zero the splat targets of both lattices for the B images of the pass (row counts are device-resident)
template <int MP>
__global__ void __launch_bounds__(kThreads)
k_mf_zero(float4 *a, const int32_t *rowbase_a, float4 *c, const int32_t *rowbase_c, int B) {
    constexpr int CH = MP / 4;
    const long long na = (long long)rowbase_a[B] * CH, nc = (long long)rowbase_c[B] * CH;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < na + nc;
         t += (long long)gridDim.x * blockDim.x) {
        if (t < na) a[t] = z; else c[t - na] = z;
    }
}

// ---------------------------------------------------------------------------------------------
// blur along one lattice axis: new = old + 0.5 (old[n1] + old[n2])  (permutohedral.cpp:556-569)
// one thread per (row, float4 chunk), rows of the pass's B images
//
// AX = 2 applies two consecutive axes (nbr, nbr + nbr_stride) in one pass without storing the
// intermediate buffer: the row's result needs the first axis' result at 3 rows, each of those at 3
// more, 9 rows of `in` in all.  Every intermediate is recomputed with the single-axis formula from the
// same operands, so the output is bit-identical to two single-axis passes; missing neighbours need no
// special case because each image's zero row points at itself on every axis.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 blur_step(float4 o, float4 a, float4 d) {
    float4 r;
    r.x = o.x + 0.5f * (a.x + d.x);
    r.y = o.y + 0.5f * (a.y + d.y);
    r.z = o.z + 0.5f * (a.z + d.z);
    r.w = o.w + 0.5f * (a.w + d.w);
    return r;
}

// one level of the neighbour tree: entry i of N becomes (its row, n1, n2) at 3i, 3i+1, 3i+2
template <int N>
__device__ __forceinline__ void blur_expand(int *u, const int2 *na) {
#pragma unroll
    for (int i = N - 1; i >= 0; i--) {
        const int2 e = na[u[i]];
        u[3 * i] = u[i];
        u[3 * i + 1] = e.x;
        u[3 * i + 2] = e.y;
    }
}

// one axis over N groups of (row, n1, n2) values, the result of group i to v[i]
template <int N>
__device__ __forceinline__ void blur_reduce(float4 *v) {
#pragma unroll
    for (int i = 0; i < N; i++) v[i] = blur_step(v[3 * i], v[3 * i + 1], v[3 * i + 2]);
}

// A pair pass over a large scattered lattice (uniform-noise images, ~176 k bilateral vertices per image) gets 64
// registers (4 CTAs per SM) so that all its row loads are in flight at once: at 32 registers (full occupancy) the 9
// loads go out in batches, each batch waits on HBM, and the pair pass cost 2.1x a single-axis pass instead of 1.65x
// (H100 SXM, 400 W).  Where the rows a pass reads mostly hit in the caches (smooth and photo-like images on the
// tile-major numbering, lattice.cu) full occupancy is faster.  The vertex counts live on the device, so a bilateral
// pair pass launches both (blur_all) and `gate` lets the one that fits run: 1 = at most kBlurCachedRows rows per
// image on average, 2 = more, 0 = always.
#ifndef DSRG_BLUR_CACHED_ROWS
#define DSRG_BLUR_CACHED_ROWS 65536
#endif
constexpr int kBlurCachedRows = DSRG_BLUR_CACHED_ROWS;
// CTAs per SM of the full-occupancy pair pass: at 32 registers ptxas spills a few bytes for MP = 4, 12 and 28, at 40
// (6 CTAs) none
__host__ __device__ constexpr int blur_cached_ctas(int mp) { return (mp == 4 || mp == 12 || mp == 28) ? 6 : 8; }
template <int MP, int AX, int CTAS>
__global__ void __launch_bounds__(kThreads, CTAS)
k_mf_blur(const float4 *in, float4 *out, const int2 *nbr, long long nbr_stride, const int32_t *rowbase, int B,
          int shared, float4 *zero, int gate) {
    constexpr int CH = MP / 4;
    constexpr int K = AX == 1 ? 3 : 9;  // rows of `in` per output row
    static_assert(AX == 1 || AX == 2, "one or two axes per pass");
    // r0 = rowbase[0] is 0.  Without it the compiler unswitches the loop on `shared` and reorders the row loads,
    // which made the bilateral blur 9 % slower on uniform-noise images (H100 SXM, 400 W)
    const long long r0 = rowbase[0], rows = rowbase[B] - r0;
    if (gate && (rows > (long long)kBlurCachedRows * B) != (gate == 2)) return;
    const int rows_img = shared ? rowbase[1] : 0;
    const long long total = rows * CH;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const long long lg = t / CH;
        const int c = (int)(t - lg * CH);
        const long long g = r0 + lg;
        // neighbour ids are image-local on the shared (spatial) lattice, global rows otherwise (rows fit an
        // int: rowbase is int32)
        const int img0 = shared ? ((int)g / rows_img) * rows_img : 0;
        // the rows whose input enters the result, expanded last axis first
        int u[K];
        u[0] = (int)g - img0;
        blur_expand<1>(u, nbr + (AX - 1) * nbr_stride);
        if constexpr (AX == 2) blur_expand<3>(u, nbr);
        const float4 *src = in + (long long)img0 * CH + c;
        float4 v[K];
#pragma unroll
        for (int i = 0; i < K; i++) v[i] = src[(size_t)(unsigned)u[i] * CH];
        // and reduced first axis first
        if constexpr (AX == 2) blur_reduce<3>(v);
        blur_reduce<1>(v);
        out[g * CH + c] = v[0];
        // the buffer that was sliced in this iteration is dead by now: clear it here so that it can be
        // the next splat target without a separate zeroing pass
        if (zero) zero[g * CH + c] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
}

// ---------------------------------------------------------------------------------------------
// exports
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_mf_export(const float *Q, float *out, int layout, int M, int N) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    for (int k = 0; k < M; k++) {
        float v = Q[((size_t)b * M + k) * N + i];
        size_t at = (layout == DSRG_LAYOUT_NCHW) ? ((size_t)b * M + k) * N + i
                                                 : ((size_t)b * N + i) * M + k;
        out[at] = v;
    }
}

// DenseCRF::currentMap (densecrf.cpp:202-211): first maximum wins
__global__ void __launch_bounds__(kThreads)
k_mf_export_map(const float *Q, int32_t *labels, int M, int N) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    int m = 0;
    float best = Q[((size_t)b * M) * N + i];
    for (int k = 1; k < M; k++) {
        float v = Q[((size_t)b * M + k) * N + i];
        if (v > best) {
            best = v;
            m = k;
        }
    }
    labels[(size_t)b * N + i] = m;
}

// result[result < min_prob] = min_prob; result /= sum (float64), pylayers.py:328-330 / :85-86;
// optional log (CRFLayer top, pylayers.py:88)
__global__ void __launch_bounds__(kThreads)
k_mf_export_renorm(const float *Q, float *result_out, float *log_out, int M, int N) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    // float64 sum in NumPy's order for the reference's layout (common.cuh:numpy_sum)
    auto clamped = [&](int k) {
        const double v = (double)Q[((size_t)b * M + k) * N + i];
        return v < 0.0001 ? 0.0001 : v;
    };
    const double s = numpy_sum<0>(clamped, M);
    for (int k = 0; k < M; k++) {
        size_t at = ((size_t)b * M + k) * N + i;
        double v = (double)Q[at];
        if (v < 0.0001) v = 0.0001;
        v = v / s;
        if (result_out) result_out[at] = (float)v;
        if (log_out) log_out[at] = (float)log(v);
    }
}

static TileLat make_tile_view(const Lattice &L, const float *val_in, float *val_out) {
    TileLat v;
    v.off = L.off;
    v.rowbase = L.rowbase;
    v.tl_nloc = L.tl_nloc;
    v.tl_hy = L.tl_hy;
    v.tl_hdr = L.tl_hdr;
    v.tl_pack = L.tl_pack;
    v.entcap = L.entcap;
    v.tl_loc = L.tl_loc;
    v.wn = L.wn;
    v.val_in = val_in;
    v.val_out = val_out;
    v.shared = L.shared;
    return v;
}

// Blur `buf` (just splatted) along all d+1 axes, two axes per pass (the spatial lattice's 3 axes run as a pair
// + a single pass, the bilateral lattice's 6 as three pairs), ping-ponging with `tmp`; returns where the result
// lives.  A pass streams its source and destination buffers through HBM (at batch 64 @ 321² each lattice's
// buffers are ~80 MB, beyond the L2), so a pair halves that traffic for 3x the row reads, most of which the
// caches serve.  On an H100 SXM at a 400 W limit the blur of a dsrg321 step went from 6.6 to 5.2 ms; one
// three-axis spatial pass (27 rows) was slower than pair + single.  Re-measured on the tile-major vertex numbering
// (lattice.cu), same card and limit: three-axis passes (spatial one pass, bilateral two, 2 CTAs per SM) took 6.1 ms
// against 4.6 for this grouping.  Bilateral pair passes pick their occupancy by the lattice's size (k_mf_blur).
template <int MP>
static float *blur_all(Engine *e, const Lattice &L, float *buf, float *tmp, float *dead, int B, int tag, int grid,
                       cudaStream_t s) {
    float *src = buf, *dst = tmp;
    for (int j = 0; j <= L.d; j += 2) {
        const float4 *in = (const float4 *)src;
        const int2 *nbr = L.nbr + (size_t)j * L.nbr_stride;
        float4 *zero = j == 0 ? (float4 *)dead : nullptr;
        if (j == L.d) {
            DSRG_LAUNCH(e, tag, s, (k_mf_blur<MP, 1, 8><<<grid, kThreads, 0, s>>>(in, (float4 *)dst, nbr, L.nbr_stride,
                                                                                L.rowbase, B, L.shared, zero, 0)));
        } else if (L.shared) {  // the spatial lattice: ~13.5 k rows per image at 321², always cached
            DSRG_LAUNCH(e, tag, s, (k_mf_blur<MP, 2, 4><<<grid, kThreads, 0, s>>>(in, (float4 *)dst, nbr, L.nbr_stride,
                                                                                L.rowbase, B, L.shared, zero, 0)));
        } else if (L.capv <= kBlurCachedRows) {  // no image of this size can have more rows
            DSRG_LAUNCH(e, tag, s, (k_mf_blur<MP, 2, blur_cached_ctas(MP)><<<grid, kThreads, 0, s>>>(
                                       in, (float4 *)dst, nbr, L.nbr_stride, L.rowbase, B, L.shared, zero, 0)));
        } else {
            DSRG_LAUNCH(e, tag, s, (k_mf_blur<MP, 2, blur_cached_ctas(MP)><<<grid, kThreads, 0, s>>>(in, (float4 *)dst, nbr, L.nbr_stride,
                                                                                L.rowbase, B, L.shared, zero, 1)));
            DSRG_LAUNCH(e, tag, s, (k_mf_blur<MP, 2, 4><<<grid, kThreads, 0, s>>>(in, (float4 *)dst, nbr, L.nbr_stride,
                                                                                L.rowbase, B, L.shared, zero, 2)));
        }
        float *t = src;
        src = dst;
        dst = t;
    }
    return src;
}

template <int MP>
static int run_impl(Engine *e, int B, const float *unary, int layout, bool clamp, float *unary_rw,
                    const dsrg_crf_params &p, cudaStream_t s) {
    const int M = e->M, N = e->N;
    dim3 gp(cdiv(N, kThreads), B);
    const int T = p.n_iters;
    // planar (NCHW) callers are read in place by the tile kernel; NHWC callers (and T == 0) go
    // through the layout-converting init kernel
    const bool direct = (layout == DSRG_LAYOUT_NCHW) && T > 0;
    const float *Usrc = direct ? unary : e->U;
    float *Urw = direct ? unary_rw : nullptr;
    const int tclamp = (direct && clamp) ? 1 : 0;
    if (!direct)
        DSRG_LAUNCH(e, T_MF_INIT, s,
                    k_mf_init<MP><<<gp, kThreads, 0, s>>>(unary, unary_rw, layout, clamp ? 1 : 0, e->U,
                                                          T == 0 ? e->Q0 : nullptr, M, N));
    e->Qcur = e->Q0;
    e->last_crf_B = B;  // host-side bookkeeping for dsrg_srg_last_crf_host (the launches below are already ordered on s)
    if (T == 0) return DSRG_OK;
    const float alpha_sp = 1.0f / (1 + powf(2, -e->sp.d));  // permutohedral.cpp:571
    const float alpha_bi = 1.0f / (1 + powf(2, -e->bi.d));
    const float c_sp = p.w2 * alpha_sp, c_bi = p.w1 * alpha_bi;
    const size_t smem = sizeof(TileSmem<MP>);
    const size_t smem_hy = sizeof(TileSmem<MP, kMaxLocHy>);
    static bool attr_done[64] = {false};   // function attributes are per device
    const int dv = e->device & 63;
    if (!attr_done[dv]) {
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_FIRST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_MID>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_LAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_FIRST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_MID>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_LAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy));
        attr_done[dv] = true;
    }
#ifndef DSRG_BLUR_GRID
#define DSRG_BLUR_GRID 8
#endif
    const int bgrid = DSRG_BLUR_GRID * e->sm_count;
    // The hybrid tiles of the batch: k_mf_tile_hy, a persistent grid over the device-resident list, issued right
    // before the plain kernel on the same stream.  A side stream (fork / join around every iteration) costs more per
    // iteration inside the replayed graph, even when the list is empty, than an empty launch in line.
    const int hgrid = DSRG_HY_CTAS * e->sm_count;
    const bool hy_on = hybrid_tiles_on(e, B);  // the same test the tile build of this pass made
    const dim3 gt(e->ntiles, B);
    // three value buffers per lattice: X = blurred values being sliced, Y = zeroed splat target,
    // Z = blur scratch
    float *spX = e->spA, *spY = e->spB, *spZ = e->spC;
    float *biX = e->biA, *biY = e->biB, *biZ = e->biC;
    DSRG_LAUNCH(e, T_MF_ZERO, s,
                k_mf_zero<MP><<<bgrid, kThreads, 0, s>>>((float4 *)spY, e->sp.rowbase, (float4 *)biY, e->bi.rowbase, B));
#define DSRG_TILE_LAUNCH(MODEV, QOUT)                                                                                 \
    do {                                                                                                              \
        if (hy_on)                                                                                                    \
            DSRG_LAUNCH(e, T_MF_TILE_HY, s,                                                                           \
                        (k_mf_tile_hy<MP, MODEV><<<hgrid, kTileThreads, smem_hy, s>>>(                                \
                            Usrc, Urw, tclamp, QOUT, vsp, vbi, c_sp, c_bi, M, N, e->W, e->H, e->tiles_x, e->ntiles,   \
                            e->tile_w, e->hy_list, e->hy_count)));                                                    \
        DSRG_LAUNCH(e, T_MF_TILE, s,                                                                                  \
                    (k_mf_tile<MP, MODEV><<<gt, kTileThreads, smem, s>>>(Usrc, Urw, tclamp, QOUT, vsp, vbi, c_sp,     \
                                                                        c_bi, M, N, e->W, e->H, e->tiles_x,           \
                                                                        e->ntiles, e->tile_w)));                      \
    } while (0)
    for (int it = 0; it <= T; it++) {
        TileLat vsp = make_tile_view(e->sp, spX, spY), vbi = make_tile_view(e->bi, biX, biY);
        if (it == T) {
            DSRG_TILE_LAUNCH(MODE_LAST, e->Q0);
            break;
        }
        if (it == 0)
            DSRG_TILE_LAUNCH(MODE_FIRST, nullptr);
        else
            DSRG_TILE_LAUNCH(MODE_MID, nullptr);
        // the old X is dead: the first blur pass clears it and it becomes the next splat target
        float *sp_res = blur_all<MP>(e, e->sp, spY, spZ, spX, B, T_MF_BLUR_SP, bgrid, s);
        float *bi_res = blur_all<MP>(e, e->bi, biY, biZ, biX, B, T_MF_BLUR_BI, bgrid, s);
        float *sp_other = (sp_res == spY) ? spZ : spY, *bi_other = (bi_res == biY) ? biZ : biY;
        float *nspY = spX, *nbiY = biX;
        spX = sp_res; spY = nspY; spZ = sp_other;
        biX = bi_res; biY = nbiY; biZ = bi_other;
    }
#undef DSRG_TILE_LAUNCH
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int meanfield_run(Engine *e, int B, const float *unary, int unary_layout, bool clamp_inplace,
                  float *unary_rw, const dsrg_crf_params &p, cudaStream_t s) {
    if (e->MP > DSRG_MAX_LABELS) return meanfield_run_wide(e, B, unary, unary_layout, clamp_inplace, unary_rw, p, s);
    switch (e->MP) {
        case 4: return run_impl<4>(e, B, unary, unary_layout, clamp_inplace, unary_rw, p, s);
        case 8: return run_impl<8>(e, B, unary, unary_layout, clamp_inplace, unary_rw, p, s);
        case 12: return run_impl<12>(e, B, unary, unary_layout, clamp_inplace, unary_rw, p, s);
        case 16: return run_impl<16>(e, B, unary, unary_layout, clamp_inplace, unary_rw, p, s);
        case 20: return run_impl<20>(e, B, unary, unary_layout, clamp_inplace, unary_rw, p, s);
        case 24: return run_impl<24>(e, B, unary, unary_layout, clamp_inplace, unary_rw, p, s);
        case 28: return run_impl<28>(e, B, unary, unary_layout, clamp_inplace, unary_rw, p, s);
        case 32: return run_impl<32>(e, B, unary, unary_layout, clamp_inplace, unary_rw, p, s);
    }
    set_error("unsupported label count %d", e->M);
    return DSRG_E_INVALID;
}

int meanfield_export(Engine *e, int B, float *out, int layout, cudaStream_t s) {
    dim3 gp(cdiv(e->N, kThreads), B);
    DSRG_LAUNCH(e, T_MF_EXPORT, s, k_mf_export<<<gp, kThreads, 0, s>>>(e->Qcur, out, layout, e->M, e->N));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int meanfield_export_map(Engine *e, int B, int32_t *labels, cudaStream_t s) {
    dim3 gp(cdiv(e->N, kThreads), B);
    DSRG_LAUNCH(e, T_MF_EXPORT, s, k_mf_export_map<<<gp, kThreads, 0, s>>>(e->Qcur, labels, e->M, e->N));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int meanfield_export_renorm(Engine *e, int B, float *result_out, float *log_out, cudaStream_t s) {
    dim3 gp(cdiv(e->N, kThreads), B);
    DSRG_LAUNCH(e, T_MF_EXPORT, s, k_mf_export_renorm<<<gp, kThreads, 0, s>>>(e->Qcur, result_out, log_out, e->M, e->N));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

}  // namespace dsrg
