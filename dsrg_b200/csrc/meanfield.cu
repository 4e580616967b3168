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
#include "simplex.cuh"
#include "kgrad.cuh"

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
    // per (pixel, r): the local vertex index and the weight wn.  k_mf_tile_bwd reads them planar ([nimg][dp1][N], tl_loc
    // and wn), the forward kernels as the tile-major blocks tl_li / tl_w ([nimg][ntiles][dp1][kTileThreads])
    const uint16_t *tl_loc;
    const float *wn;
    const float *val_in;     // blurred values of the previous splat (slice source)
    float *val_out;          // zeroed values (splat target)
    int entcap;
    int shared;
};

// MODE & 3 is the iteration's place in the loop.  MODE_HIST (the training forward, dsrg_crf_forward_train_dev) also
// stores every iteration's Q_t to the caller's history for the backward, never clamps the unary, and reads the Potts
// weights from device memory when the U_rw argument (unused without the clamp) carries them: {w1, w2}, with c_sp /
// c_bi then passed as alpha alone.  Without MODE_HIST the instantiations are the inference kernels, unchanged.
// MODE_COMPAT (with MODE_HIST: dsrg_crf_forward_train_compat_dev; without it: the learned inference,
// dsrg_crf_batch_learned_dev, storing Q_T alone; in k_mf_tile_bwd: dsrg_crf_backward_compat_dev) replaces the Potts
// messages by label-compatibility matrices, t = U - mu_sp F_sp(Q) - mu_bi F_bi(Q): U_rw (potts in the backward) then
// carries {mu_bi, mu_sp} ([2][M][M], row l = the message to label l), c_sp / c_bi are alpha alone.  The tile kernels
// write U_rw only in the clamp of a MODE_FIRST inference instantiation, and MODE_COMPAT has no MODE_FIRST there (the
// first iteration slices nothing and runs the Potts kernel), so the matrices are never written.
enum { MODE_FIRST = 0, MODE_MID = 1, MODE_LAST = 2, MODE_HIST = 4, MODE_COMPAT = 8, MODE_GSTORE = 16 };

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

// The forward kernels' shared memory: the weight blocks of the tile (tiles.cu) are bulk-copied into wtab, its local-index
// blocks into loc, both [r][thread]; a thread reads its own slot of each row, so the slice is free of bank conflicts
template <int MP, int MAXBI = kMaxLocBi>
struct TileSmemFwd {
    static_assert(sizeof(TileStage<MP, MAXBI>) % 16 == 0, "wtab's rows are bulk-copy destinations");
    TileSmem<MP, MAXBI> t;
    alignas(16) uint16_t loc[kEntRows * kTileThreads];
};

// the size of a lattice's CSR entry block as bulk-copied, from the header of its last segment
__device__ __forceinline__ uint32_t ent_block_bytes(int2 last) {
    return ((uint32_t)((last.x & 0xffff) + (((last.x >> 16) + 1) & ~1)) * 2u + 15u) & ~15u;
}

// the current tile's weights into the table its CSR entries index (k_mf_tile_bwd; the forward kernels bulk-copy the
// tile's tl_w blocks there); the CTA's thread t is the tile's pixel t
__device__ __forceinline__ void tile_put_weights(float *wtab, const float *w_sp, const float *w_bi) {
#pragma unroll
    for (int r = 0; r < 3; r++) wtab[(ent_r0(3) + r) * kTileThreads + threadIdx.x] = w_sp[r];
#pragma unroll
    for (int r = 0; r < 6; r++) wtab[(ent_r0(6) + r) * kTileThreads + threadIdx.x] = w_bi[r];
}

// A pixel's weight and local vertex index at incidence r.  k_mf_tile_bwd holds the weights in registers and reads the
// indices from the planar tl_loc, `stride` apart; the forward kernels (SW) read both from their shared tables, rows
// kTileThreads apart, w and loc pointing at the thread's own slot of row 0.
template <bool SW>
__device__ __forceinline__ float w_at(const float *w, int r) { return w[SW ? r * kTileThreads : r]; }
template <bool SW>
__device__ __forceinline__ int loc_at(const uint16_t *loc, size_t stride, int r) {
    return SW ? (int)loc[r * kTileThreads] : (int)__ldg(loc + r * stride);
}

// slice one lattice from the staged rows (shared memory): t += coef * sum_r wn_r * row_r
// tail1: M = MP - 3 (e.g. 21 labels in 24 lanes): the last chunk holds ONE real channel, so a 32-bit load
// (one shared-memory wavefront per warp) replaces the 128-bit one (four)
template <int MP, int DP1, bool SW = false>
__device__ __forceinline__ void tile_slice_smem(const float4 *vs, const uint16_t *loc, size_t stride,
                                                const float *w, float coef, float *t, bool tail1) {
    constexpr int CH = MP / 4, CHP = TileRow<MP>::CHP;
#pragma unroll
    for (int r = 0; r < DP1; r++) {
        const float4 *row = vs + loc_at<SW>(loc, stride, r) * CHP;
        const float wr = coef * w_at<SW>(w, r);
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
template <int MP, int DP1, bool SW = false>
__device__ __forceinline__ void tile_slice_global(const float4 *vin, const int32_t *off, size_t stride,
                                                  int base, const float *w, float coef, float *t) {
    constexpr int CH = MP / 4;
#pragma unroll
    for (int r = 0; r < DP1; r++) {
        const float4 *row = vin + (size_t)(base + off[r * stride]) * CH;
        const float wr = coef * w_at<SW>(w, r);
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
template <int MP, int DP1, bool SW = false>
__device__ __forceinline__ unsigned tile_slice_mixed(const float4 *vs, const uint16_t *loc, const float4 *vin,
                                                     const int32_t *off, size_t stride, int base, const float *w,
                                                     float coef, float *t) {
    constexpr int CH = MP / 4, CHP = TileRow<MP>::CHP;
    unsigned remote = 0;  // bit r: incidence r of this pixel goes direct
#pragma unroll
    for (int r = 0; r < DP1; r++) {
        const int l = loc_at<SW>(loc, stride, r);
        const float wr = coef * w_at<SW>(w, r);
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
template <int DP1, bool SW = false>
__device__ __forceinline__ unsigned tile_remote_mask(const uint16_t *loc, size_t stride) {
    unsigned remote = 0;
#pragma unroll
    for (int r = 0; r < DP1; r++)
        if (loc_at<SW>(loc, stride, r) == kLocRemote) remote |= 1u << r;
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
template <int MP, int DP1, bool SW = false>
__device__ __forceinline__ void tile_splat_direct(float4 *vout, const int32_t *off, size_t stride,
                                                  int base, const float *w, const float *q) {
    constexpr int CH = MP / 4;
#pragma unroll
    for (int r = 0; r < DP1; r++) {
        float4 *row = vout + (size_t)(base + off[r * stride]) * CH;
        const float wr = w_at<SW>(w, r);
#pragma unroll
        for (int c = 0; c < CH; c++)
            atomicAdd(row + c, make_float4(wr * q[4 * c], wr * q[4 * c + 1], wr * q[4 * c + 2], wr * q[4 * c + 3]));
    }
}

// direct splat of one pixel's remote incidences (hybrid tiles): MP/4 vector reductions per such row
template <int MP, int DP1, bool SW = false>
__device__ __forceinline__ void tile_splat_remote(float4 *vout, unsigned remote, const int32_t *off, size_t stride,
                                                  int base, const float *w, const float *q) {
    constexpr int CH = MP / 4;
#pragma unroll
    for (int r = 0; r < DP1; r++) {
        if (!(remote >> r & 1u)) continue;
        float4 *row = vout + (size_t)(base + __ldg(off + r * stride)) * CH;
        const float wr = w_at<SW>(w, r);
#pragma unroll
        for (int c = 0; c < CH; c++)
            atomicAdd(row + c, make_float4(wr * q[4 * c], wr * q[4 * c + 1], wr * q[4 * c + 2], wr * q[4 * c + 3]));
    }
}

// ---- label-compatibility matrices (MODE_COMPAT) ----
// They sit in dynamic shared memory behind the kernel's TileSmem, zero-padded to [2][MP][MP] ({bi, sp}); every
// thread of a warp reads the same element, so the reads are broadcasts.  The CTA stages them before its first barrier.
template <int MP>
constexpr size_t kCompatSmem = sizeof(float) * 2 * MP * MP;
template <int MP>
__device__ __forceinline__ const float *compat_stage(unsigned char *at, const float *mu, int M) {
    float *s = reinterpret_cast<float *>(at);
    for (int i = threadIdx.x; i < 2 * MP * MP; i += kTileThreads) {
        const int k = i / (MP * MP), l = i / MP % MP, l2 = i % MP;
        s[i] = (l < M && l2 < M) ? __ldg(mu + ((size_t)k * M + l) * M + l2) : 0.0f;
    }
    return s;
}

// The phantom lanes of a slice are set to zero: under tail1 the slice never reads them, elsewhere they hold whatever the
// staged or global rows hold there, and the zero-padded columns of mu would turn a non-finite one into NaN (0 * inf).
template <int MP>
__device__ __forceinline__ void compat_clear_phantoms(float *sl, int M) {
#pragma unroll
    for (int k = 0; k < MP; k++)
        if (k >= M) sl[k] = 0.0f;
}

// t -= mu sl (the forward's message) or, with TRANSPOSE, t -= mu^T sl (the backward's G_t), as fma chains over the
// labels in ascending order.  The empty asm keeps each row's loads of mu next to that row's fmas, so that the
// registers hold one row of mu at a time beside t and the slice.
template <int MP, bool TRANSPOSE>
__device__ __forceinline__ void compat_apply(const float *mu, const float *sl, float *t) {
#pragma unroll
    for (int l = 0; l < MP; l++) {
#pragma unroll
        for (int l2 = 0; l2 < MP; l2++) t[l] = fmaf(-mu[TRANSPOSE ? l2 * MP + l : l * MP + l2], sl[l2], t[l]);
        asm volatile("" ::: "memory");
    }
}

// tile_slice_smem / tile_slice_global one row at a time (the same fma chain): at 32 labels ptxas otherwise issued a
// whole lattice's row loads ahead of the previous lattice's message and spilled.  w and loc are the shared tables (SW).
template <int MP, int DP1>
__device__ __forceinline__ void compat_slice(bool direct, const float4 *vs, const uint16_t *loc, const float4 *vin,
                                             const int32_t *off, size_t stride, int base, const float *w, float coef,
                                             float *sl, bool tail1) {
#pragma unroll
    for (int r = 0; r < DP1; r++) {
        if (!direct)
            tile_slice_smem<MP, 1, true>(vs, loc + r * kTileThreads, stride, w + r * kTileThreads, coef, sl, tail1);
        else
            tile_slice_global<MP, 1, true>(vin, off + r * stride, stride, base, w + r * kTileThreads, coef, sl);
        asm volatile("" ::: "memory");
    }
}

// ---- the per-tile steps both tile kernels share ----
// The tile coordinates and the bulk-copy staging are still written out in each kernel: moved into a shared helper,
// either one changed the SASS of some k_mf_tile / k_mf_tile_hy instantiations (register choice, loop offsets).
//
// Park the pixel's Q row in the staging buffer (once every thread is done reading the staged rows) and, with PUT_W
// (k_mf_tile_bwd: the forward kernels bulk-copy theirs), its weights in wtab, for the CSR splat; returns the Q rows
template <int MP, int MAXBI, bool PUT_W = true>
__device__ __forceinline__ const float4 *tile_park(TileSmem<MP, MAXBI> &smt, const float *t, const float *w_sp,
                                                   const float *w_bi) {
    constexpr int CH = MP / 4, CHP = TileStage<MP, MAXBI>::CHP;
    const int tid = threadIdx.x;
    __syncthreads();
    float4 *qs = smt.st.buf;
#pragma unroll
    for (int c = 0; c < CH; c++) qs[tid * CHP + c] = make_float4(t[4 * c], t[4 * c + 1], t[4 * c + 2], t[4 * c + 3]);
    if (PUT_W) tile_put_weights(smt.wtab, w_sp, w_bi);
    __syncthreads();
    return qs;
}

// The forward kernels' per-tile blocks (tiles.cu), as ONE arrival on the tile's barrier: both weight blocks (the slice
// and every splat read them) into wtab and, where the slice reads them (li_*), the local-index blocks into loc
template <int MP, int MAXBI>
__device__ __forceinline__ void tile_fetch_blocks(TileSmemFwd<MP, MAXBI> &smf, const TileLat &sp, const TileLat &bi,
                                                  size_t ti_sp, size_t ti_bi, bool li_sp, bool li_bi) {
    constexpr uint32_t kSp = 3 * kTileThreads, kBi = 6 * kTileThreads;  // slots per block
    uint64_t *bar = &smf.t.st.bar;
    mbar_arrive_expect_tx(bar, (kSp + kBi) * 4u + (li_sp ? kSp * 2u : 0u) + (li_bi ? kBi * 2u : 0u));
    bulk_g2s(smf.t.wtab + ent_r0(3) * kTileThreads, sp.wn + ti_sp * kSp, kSp * 4u, bar);
    bulk_g2s(smf.t.wtab + ent_r0(6) * kTileThreads, bi.wn + ti_bi * kBi, kBi * 4u, bar);
    if (li_sp) bulk_g2s(smf.loc + ent_r0(3) * kTileThreads, sp.tl_loc + ti_sp * kSp, kSp * 2u, bar);
    if (li_bi) bulk_g2s(smf.loc + ent_r0(6) * kTileThreads, bi.tl_loc + ti_bi * kBi, kBi * 2u, bar);
}

// Q = softmax(t) in place (expAndNormalize, densecrf.cpp:98-106); the last iteration (every one with MODE_HIST) stores
// it to Qout
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
    if ((MODE & 3) == MODE_LAST || (MODE & MODE_HIST)) {
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

// The pixel's unaries into t (zeros outside the image).  U is either the engine's planar copy or, for NCHW callers,
// the caller's buffer itself; the reference's in-place clamp (pylayers.py:312) is then applied on the fly and written
// back once, by the first iteration.
template <int MP, int MODE>
__device__ __forceinline__ void tile_load_pixel(const float *U, float *U_rw, int clamp, int M, int N, int b, int pix,
                                                bool in, float *t) {
    {
        const size_t ub = (size_t)b * M * N + pix;
        const float *Ub = U + ub;
#pragma unroll
        for (int k = 0; k < MP; k++) {
            float v = 0.0f;
            if (in && k < M) v = ((MODE & 3) == MODE_FIRST) ? *Ub : __ldg(Ub);  // read-only path once nothing writes U
            if ((MODE & 3) == MODE_FIRST && !(MODE & MODE_HIST)) {  // later iterations read the values this one wrote back
                if (clamp && in && k < M && v < kMinProb) {
                    v = kMinProb;
                    U_rw[ub + (size_t)k * N] = v;
                }
            }
            t[k] = v;
            Ub += N;
        }
    }
}

// MODE_COMPAT holds a slice beside t (2 MP floats): like k_mf_tile_bwd it runs one CTA per SM above 12 labels rather
// than spill
template <int MP, int MODE>
__global__ void __launch_bounds__(kTileThreads, (MODE & MODE_COMPAT) ? (MP > 12 ? 1 : 2) : DSRG_TILE_CTAS)
k_mf_tile(const float *U, float *U_rw, int clamp, float *__restrict__ Qout, TileLat sp, TileLat bi, float c_sp,
          float c_bi, int M, int N, int W, int H, int tiles_x, int ntiles, int tile_w) {
    static_assert(!(MODE & MODE_COMPAT) || (MODE & 3) != MODE_FIRST, "U_rw carries the matrices: nothing may clamp");
    constexpr int kRowBytes = MP * 4;
    using SF = TileSmemFwd<MP>;
    using ST = TileStage<MP>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    SF &smf = *reinterpret_cast<SF *>(smem_raw);
    TileSmem<MP> &smt = smf.t;
    ST &sm = smt.st;
    // A hybrid tile is k_mf_tile_hy's.  The test reads a byte map of its own and stands before anything else: the
    // same test on the tile's vertex count, wherever it was placed, made ptxas allocate this kernel's 64 registers
    // differently (more spill traffic in the splat loop, also on images that have no such tile at all).
    if (bi.tl_hy[(size_t)blockIdx.y * ntiles + blockIdx.x]) return;
    const float *mu = nullptr;
    if constexpr ((MODE & MODE_COMPAT) != 0) {
        mu = compat_stage<MP>(smem_raw + sizeof(SF), U_rw, M);
    } else if ((MODE & MODE_HIST) && U_rw) {
        c_sp *= __ldg(U_rw + 1);
        c_bi *= __ldg(U_rw);
    }
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

    // ---- asynchronous staging: every local vertex's value row (96 B), the two CSR entry blocks and the tile's weight
    // and local-index blocks are pulled into shared memory by the bulk-copy engine while the threads load their unaries
    const int n_copies = ((MODE & 3) != MODE_FIRST ? n_sp + n_bi : 0) + ((MODE & 3) != MODE_LAST ? (n_sp > 0) + (n_bi > 0) : 0);
    if (tid == 0) {
        mbar_init(&sm.bar, n_copies + 1);
        smt.wtab[kEntZero] = 0.0f;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (tid == kTileThreads - 1)  // the last thread stages a vertex only when the tile has more than 256
        tile_fetch_blocks(smf, sp, bi, ti_sp, ti_bi, (MODE & 3) != MODE_FIRST && !fb_sp, (MODE & 3) != MODE_FIRST && !fb_bi);
    for (int i = tid; i < n_sp + n_bi; i += kTileThreads) {  // up to kMaxLocSp + kMaxLocBi local vertices
        const bool is_sp = i < n_sp;
        const int lv = is_sp ? i : i - n_sp;
        const int2 h = __ldg((is_sp ? hdr_sp : hdr_bi) + lv);
        const int row = (is_sp ? base_sp : base_bi) + h.y;
        if ((MODE & 3) != MODE_FIRST) {
            mbar_arrive_expect_tx(&sm.bar, kRowBytes);
            bulk_g2s((is_sp ? vs_sp : vs_bi) + lv * CHP, (is_sp ? sp.val_in : bi.val_in) + (size_t)row * MP,
                     kRowBytes, &sm.bar);
        }
        if ((MODE & 3) != MODE_LAST && lv == (is_sp ? n_sp : n_bi) - 1) {  // the last segment tells the block's length
            const uint32_t bytes = ent_block_bytes(h);
            mbar_arrive_expect_tx(&sm.bar, bytes);
            bulk_g2s(is_sp ? ent_sp : ent_bi,
                     is_sp ? sp.tl_pack + ti_sp * sp.entcap : bi.tl_pack + ti_bi * bi.entcap, bytes, &sm.bar);
        }
    }

    // ---- per-pixel data (thread = pixel); its weights and local indices are its slots of the shared tables ----
    float t[MP];
    tile_load_pixel<MP, MODE>(U, U_rw, clamp, M, N, b, pix, in, t);
    const float *w_sp = smt.wtab + ent_r0(3) * kTileThreads + tid, *w_bi = smt.wtab + ent_r0(6) * kTileThreads + tid;
    const uint16_t *loc_sp = smf.loc + ent_r0(3) * kTileThreads + tid, *loc_bi = smf.loc + ent_r0(6) * kTileThreads + tid;
    mbar_wait(&sm.bar, 0);

    // ---- slice + update ----
#ifdef DSRG_NO_TAIL1
    const bool tail1 = false;
#else
    const bool tail1 = (M == MP - 3);
#endif
    if ((MODE & 3) != MODE_FIRST && in) {
        if constexpr ((MODE & MODE_COMPAT) != 0) {
            // each lattice sliced into its own vector, then its matrix message
            float sl[MP];
#pragma unroll
            for (int k = 0; k < MP; k++) sl[k] = 0.0f;
            compat_slice<MP, 3>(fb_sp, vs_sp, loc_sp, reinterpret_cast<const float4 *>(sp.val_in), sp.off + px_sp,
                                strideN, base_sp, w_sp, c_sp, sl, tail1);
            compat_clear_phantoms<MP>(sl, M);
            compat_apply<MP, false>(mu + MP * MP, sl, t);
#pragma unroll
            for (int k = 0; k < MP; k++) sl[k] = 0.0f;
            compat_slice<MP, 6>(fb_bi, vs_bi, loc_bi, reinterpret_cast<const float4 *>(bi.val_in), bi.off + px_bi,
                                strideN, base_bi, w_bi, c_bi, sl, tail1);
            compat_clear_phantoms<MP>(sl, M);
            compat_apply<MP, false>(mu, sl, t);
        } else {
            if (!fb_sp)
                tile_slice_smem<MP, 3, true>(vs_sp, loc_sp, strideN, w_sp, c_sp, t, tail1);
            else
                tile_slice_global<MP, 3, true>(reinterpret_cast<const float4 *>(sp.val_in), sp.off + px_sp, strideN,
                                               base_sp, w_sp, c_sp, t);
            if (!fb_bi)
                tile_slice_smem<MP, 6, true>(vs_bi, loc_bi, strideN, w_bi, c_bi, t, tail1);
            else
                tile_slice_global<MP, 6, true>(reinterpret_cast<const float4 *>(bi.val_in), bi.off + px_bi, strideN,
                                               base_bi, w_bi, c_bi, t);
        }
    }
    tile_update<MP, MODE>(t, M, N, Qout, b, pix, in);
    if ((MODE & 3) == MODE_LAST) return;
    const float4 *qs = tile_park<MP, kMaxLocBi, false>(smt, t, nullptr, nullptr);
    // ---- splat ----
    float4 *vout_sp = reinterpret_cast<float4 *>(sp.val_out), *vout_bi = reinterpret_cast<float4 *>(bi.val_out);
    if (fb_sp && in) tile_splat_direct<MP, 3, true>(vout_sp, sp.off + px_sp, strideN, base_sp, w_sp, t);
    if (fb_bi && in) tile_splat_direct<MP, 6, true>(vout_bi, bi.off + px_bi, strideN, base_bi, w_bi, t);
    tile_splat_csr<MP>(vout_sp, vout_bi, n_sp, n_bi, hdr_sp, hdr_bi, base_sp, base_bi, ent_sp, ent_bi, qs, smt.wtab);
}

// Hybrid tiles (tiles.cu: more distinct vertices than the shared-memory path of k_mf_tile holds -- textured images,
// whose vertices are shared in colour space rather than between neighbouring pixels).  A persistent grid walks the
// list of such tiles: the kMaxLocHy most-touched vertices of a tile go through shared memory exactly like in
// k_mf_tile (bulk-copied rows, CSR splat), the remaining incidences are sliced from and reduced into global
// memory straight from the registers.  Its own register / shared-memory budget (DSRG_HY_CTAS CTAs per SM) keeps
// this code out of k_mf_tile's 64-register allocation.
template <int MP, int MODE>
__global__ void __launch_bounds__(kTileThreads, (MODE & MODE_COMPAT) ? (MP > 12 ? 1 : 2) : DSRG_HY_CTAS)
k_mf_tile_hy(const float *U, float *U_rw, int clamp, float *__restrict__ Qout, TileLat sp, TileLat bi, float c_sp,
             float c_bi, int M, int N, int W, int H, int tiles_x, int ntiles, int tile_w, const int2 *hy_list,
             const int *hy_count) {
    static_assert(!(MODE & MODE_COMPAT) || (MODE & 3) != MODE_FIRST, "U_rw carries the matrices: nothing may clamp");
    constexpr int kRowBytes = MP * 4;
    using ST = TileStage<MP, kMaxLocHy>;
    using SF = TileSmemFwd<MP, kMaxLocHy>;
    constexpr int CHP = ST::CHP;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    SF &smf = *reinterpret_cast<SF *>(smem_raw);
    TileSmem<MP, kMaxLocHy> &smt = smf.t;
    ST &sm = smt.st;
    const int tid = threadIdx.x;
    const int nhy = *hy_count;
    const float *mu = nullptr;   // visible after the first tile's barriers
    if constexpr ((MODE & MODE_COMPAT) != 0) {
        mu = compat_stage<MP>(smem_raw + sizeof(SF), U_rw, M);
    } else if ((MODE & MODE_HIST) && U_rw) {
        c_sp *= __ldg(U_rw + 1);
        c_bi *= __ldg(U_rw);
    }
    const size_t strideN = (size_t)N;
    float4 *vs_sp = sm.buf, *vs_bi = sm.buf + kMaxLocSp * CHP;
    uint16_t *ent_sp = sm.ent, *ent_bi = sm.ent + ST::kEntSp;
    if (tid == 0) smt.wtab[kEntZero] = 0.0f;  // visible after the first tile's barriers
    const float *w_sp = smt.wtab + ent_r0(3) * kTileThreads + tid, *w_bi = smt.wtab + ent_r0(6) * kTileThreads + tid;
    const uint16_t *loc_sp = smf.loc + ent_r0(3) * kTileThreads + tid, *loc_bi = smf.loc + ent_r0(6) * kTileThreads + tid;
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

        // ---- asynchronous staging of the local vertices' rows, the CSR entry blocks and the tile's weight and
        // local-index blocks (as in k_mf_tile; every incidence of the bilateral lattice may be remote) ----
        const int n_copies = ((MODE & 3) != MODE_FIRST ? n_sp + n_bi : 0) + ((MODE & 3) != MODE_LAST ? (n_sp > 0) + (n_bi > 0) : 0);
        if (tid == 0) {
            mbar_init(&sm.bar, n_copies + 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        // the previous tile of this CTA wrote its Q rows into the same shared memory through the generic proxy: order
        // those writes before the bulk copies (async proxy) of this tile
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (tid == kTileThreads - 1)
            tile_fetch_blocks(smf, sp, bi, ti_sp, ti_bi, (MODE & 3) != MODE_FIRST || hy_sp, true);
        for (int i = tid; i < n_sp + n_bi; i += kTileThreads) {
            const bool is_sp = i < n_sp;
            const int lv = is_sp ? i : i - n_sp;
            const int2 h = __ldg((is_sp ? hdr_sp : hdr_bi) + lv);
            const int row = (is_sp ? base_sp : base_bi) + h.y;
            if ((MODE & 3) != MODE_FIRST) {
                mbar_arrive_expect_tx(&sm.bar, kRowBytes);
                bulk_g2s((is_sp ? vs_sp : vs_bi) + lv * CHP, (is_sp ? sp.val_in : bi.val_in) + (size_t)row * MP,
                         kRowBytes, &sm.bar);
            }
            if ((MODE & 3) != MODE_LAST && lv == (is_sp ? n_sp : n_bi) - 1) {  // the last segment tells the block's length
                const uint32_t bytes = ent_block_bytes(h);
                mbar_arrive_expect_tx(&sm.bar, bytes);
                bulk_g2s(is_sp ? ent_sp : ent_bi,
                         is_sp ? sp.tl_pack + ti_sp * sp.entcap : bi.tl_pack + ti_bi * bi.entcap, bytes, &sm.bar);
            }
        }

        // ---- per-pixel data ----
        float t[MP];
        tile_load_pixel<MP, MODE>(U, U_rw, clamp, M, N, b, pix, in, t);
        mbar_wait(&sm.bar, 0);

        // ---- slice + update ----
        unsigned rm_sp = 0, rm_bi = 0;  // this pixel's incidences that go direct
        if (in) {
            if ((MODE & 3) != MODE_FIRST && (MODE & MODE_COMPAT)) {
                float sl[MP];
#pragma unroll
                for (int k = 0; k < MP; k++) sl[k] = 0.0f;
                rm_sp = tile_slice_mixed<MP, 3, true>(vs_sp, loc_sp, reinterpret_cast<const float4 *>(sp.val_in),
                                                      sp.off + px_sp, strideN, base_sp, w_sp, c_sp, sl);
                compat_clear_phantoms<MP>(sl, M);
                compat_apply<MP, false>(mu + MP * MP, sl, t);
#pragma unroll
                for (int k = 0; k < MP; k++) sl[k] = 0.0f;
                rm_bi = tile_slice_mixed<MP, 6, true>(vs_bi, loc_bi, reinterpret_cast<const float4 *>(bi.val_in),
                                                      bi.off + px_bi, strideN, base_bi, w_bi, c_bi, sl);
                compat_clear_phantoms<MP>(sl, M);
                compat_apply<MP, false>(mu, sl, t);
            } else if ((MODE & 3) != MODE_FIRST) {
                rm_sp = tile_slice_mixed<MP, 3, true>(vs_sp, loc_sp, reinterpret_cast<const float4 *>(sp.val_in),
                                                      sp.off + px_sp, strideN, base_sp, w_sp, c_sp, t);
                rm_bi = tile_slice_mixed<MP, 6, true>(vs_bi, loc_bi, reinterpret_cast<const float4 *>(bi.val_in),
                                                      bi.off + px_bi, strideN, base_bi, w_bi, c_bi, t);
            } else {
                if (hy_sp) rm_sp = tile_remote_mask<3, true>(loc_sp, strideN);
                if (hy_bi) rm_bi = tile_remote_mask<6, true>(loc_bi, strideN);
            }
        }
        tile_update<MP, MODE>(t, M, N, Qout, b, pix, in);
        if ((MODE & 3) != MODE_LAST) {
            // ---- splat: remote incidences straight from the registers, the local vertices through the CSR ----
            if (rm_sp) tile_splat_remote<MP, 3, true>(vout_sp, rm_sp, sp.off + px_sp, strideN, base_sp, w_sp, t);
            if (rm_bi) tile_splat_remote<MP, 6, true>(vout_bi, rm_bi, bi.off + px_bi, strideN, base_bi, w_bi, t);
            const float4 *qs = tile_park<MP, kMaxLocHy, false>(smt, t, nullptr, nullptr);
            tile_splat_csr<MP>(vout_sp, vout_bi, n_sp, n_bi, hdr_sp, hdr_bi, base_sp, base_bi, ent_sp, ent_bi, qs,
                               smt.wtab);
        }
        __syncthreads();  // the tile is done with the shared buffers and the barrier
        if (tid == 0) asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(smem_u32(&sm.bar)) : "memory");
    }
}

// ---------------------------------------------------------------------------------------------
// The backward of the mean field (DenseCRF::gradient, densecrf.cpp:238-297), one launch per iteration, run from T
// down to 0 on the forward's tile-local views.  With G = dL/dQ_T and F(X) = norm K(norm X) (alpha folded in):
//   FIRST : g_T = Q_T (G - <G, Q_T>);  grad_U = g_T;  splat wn g_T
//   MID   : S_sp = F_sp^T(g_{t+1}), S_bi = F_bi^T(g_{t+1})   (slice of the reverse-blurred splat)
//           dL/dw2 += <S_sp, Q_t>, dL/dw1 += <S_bi, Q_t>;  G_t = w2 S_sp + w1 S_bi
//           g_t = Q_t (G_t - <G_t, Q_t>);  grad_U += g_t;  splat wn g_t
//   LAST  : MID without the splat (t = 0)
// F^T is the same splat and slice around the transposed blur (blur_all with reverse), so only the blur differs from
// the forward.  The Potts terms use <g, F(Q)> = <F^T(g), Q>, which needs no forward filter of Q_t (the reference
// filters Q_t, pairwise.cpp:190-195: equal in exact arithmetic).  Each thread owns its pixel's grad_U row; each CTA
// adds its tile's two Potts partials to part[b][tile] (FIRST writes zeros), so the sums are deterministic.
// Every tile kind runs here: hybrid tiles take the direct global path for the bilateral lattice, like overflow tiles.
// A pixel holds Q_t, G_t and one slice (3 MP floats): above 12 labels that takes more than 128 registers, so those
// instantiations run one CTA per SM rather than spill (MODE_COMPAT: above 8, for its outer products).
//
// MODE_COMPAT (potts = {mu_bi, mu_sp}, part = the [B][ntiles][2][M][M] float partials): G_t = -(mu_sp^T S_sp +
// mu_bi^T S_bi), and dL/dmu_k += -sum_i S_k,i (x) Q_t,i, again by <g, F(Q)> = <F^T(g), Q> per label pair.  Each pixel
// parks S_bi, S_sp and Q_t in shared memory (behind mu, rows of an odd stride so that the parking is conflict free);
// after the splat each thread owns fixed (l, l') entries and sums them over the tile's pixels in pixel order.
//
// MODE_GSTORE (the kernel-bandwidth backward) also stores g_t, the vector the launch splats, to gstore ([B][M][N]):
// k_kg_pass of iteration t - 1 reads it before the next launch overwrites it.
// ---------------------------------------------------------------------------------------------
// rows of the parked S_bi / S_sp / Q_t: an odd stride >= M
__host__ __device__ constexpr int compat_park_stride(int m) { return m | 1; }
template <int MP>
constexpr size_t kCompatParkSmem = sizeof(float) * 3 * kTileThreads * compat_park_stride(MP);

template <int MP, int MODE>
__global__ void __launch_bounds__(kTileThreads, MP > ((MODE & MODE_COMPAT) ? 8 : 12) ? 1 : 2)
k_mf_tile_bwd(const float *__restrict__ G, const float *__restrict__ Qt, float *__restrict__ gU, TileLat sp,
              TileLat bi, float a_sp, float a_bi, const float *potts, float w1, float w2, float2 *part, int M, int N,
              int W, int H, int tiles_x, int ntiles, int tile_w, float *gstore) {
    constexpr int kRowBytes = MP * 4;
    constexpr int PH = MODE & 3;   // the iteration's place in the loop
    constexpr bool kCompat = (MODE & MODE_COMPAT) != 0;
    using SM = TileSmem<MP>;
    using ST = TileStage<MP>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ float2 red[kTileThreads / 32];
    SM &smt = *reinterpret_cast<SM *>(smem_raw);
    ST &sm = smt.st;
    const int tile = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const float *mu = nullptr;
    float *park = nullptr;
    if constexpr (kCompat) {
        mu = compat_stage<MP>(smem_raw + sizeof(SM), potts, M);
        park = reinterpret_cast<float *>(smem_raw + sizeof(SM) + kCompatSmem<MP>);
    } else if (potts) {
        w1 = __ldg(potts);
        w2 = __ldg(potts + 1);
    }
    const int tx = tile % tiles_x, ty = tile / tiles_x;
    const int x = tx * tile_w + (tid & 31), y = ty * kTileH + (tid >> 5);
    const bool in = (tid & 31) < tile_w && x < W && y < H;
    const int pix = in ? y * W + x : 0;
    const int sb_sp = sp.shared ? 0 : b, sb_bi = bi.shared ? 0 : b;
    const size_t ti_sp = (size_t)sb_sp * ntiles + tile, ti_bi = (size_t)sb_bi * ntiles + tile;
    const int nl_sp = sp.tl_nloc[ti_sp], nl_bi = bi.tl_nloc[ti_bi];
    const bool fb_sp = nl_sp < 0, fb_bi = nl_bi < 0 || bi.tl_hy[ti_bi];
    const int n_sp = fb_sp ? 0 : nl_sp, n_bi = fb_bi ? 0 : nl_bi;
    const int base_sp = sp.rowbase[b], base_bi = bi.rowbase[b];
    constexpr int CHP = ST::CHP;
    float4 *vs_sp = sm.buf, *vs_bi = sm.buf + kMaxLocSp * CHP;
    const int2 *hdr_sp = sp.tl_hdr + ti_sp * kMaxLocSp, *hdr_bi = bi.tl_hdr + ti_bi * kMaxLocHy;
    uint16_t *ent_sp = sm.ent, *ent_bi = sm.ent + ST::kEntSp;
    const size_t strideN = (size_t)N;
    const size_t px_sp = (size_t)sb_sp * 3 * N + pix, px_bi = (size_t)sb_bi * 6 * N + pix;

    // ---- asynchronous staging, as in k_mf_tile ----
    const int n_copies = (PH != MODE_FIRST ? n_sp + n_bi : 0) + (PH != MODE_LAST ? (n_sp > 0) + (n_bi > 0) : 0);
    if (tid == 0) {
        mbar_init(&sm.bar, n_copies > 0 ? n_copies : 1);
        smt.wtab[kEntZero] = 0.0f;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    for (int i = tid; i < n_sp + n_bi; i += kTileThreads) {
        const bool is_sp = i < n_sp;
        const int lv = is_sp ? i : i - n_sp;
        const int2 h = __ldg((is_sp ? hdr_sp : hdr_bi) + lv);
        const int row = (is_sp ? base_sp : base_bi) + h.y;
        if (PH != MODE_FIRST) {
            mbar_arrive_expect_tx(&sm.bar, kRowBytes);
            bulk_g2s((is_sp ? vs_sp : vs_bi) + lv * CHP, (is_sp ? sp.val_in : bi.val_in) + (size_t)row * MP,
                     kRowBytes, &sm.bar);
        }
        if (PH != MODE_LAST && lv == (is_sp ? n_sp : n_bi) - 1) {
            const uint32_t bytes = ent_block_bytes(h);
            mbar_arrive_expect_tx(&sm.bar, bytes);
            bulk_g2s(is_sp ? ent_sp : ent_bi,
                     is_sp ? sp.tl_pack + ti_sp * sp.entcap : bi.tl_pack + ti_bi * bi.entcap, bytes, &sm.bar);
        }
    }
    if (n_copies == 0 && tid == 0) mbar_arrive_expect_tx(&sm.bar, 0);

    // ---- per-pixel data: Q_t, the weights, and G (FIRST) ----
    const size_t ub = (size_t)b * M * N + pix;
    float q[MP], t[MP], w_sp[3], w_bi[6];
#pragma unroll
    for (int k = 0; k < MP; k++) {
        q[k] = (in && k < M) ? __ldg(Qt + ub + (size_t)k * N) : 0.0f;
        t[k] = (PH == MODE_FIRST && in && k < M) ? __ldg(G + ub + (size_t)k * N) : 0.0f;
    }
#pragma unroll
    for (int r = 0; r < 3; r++) w_sp[r] = in ? __ldg(sp.wn + px_sp + r * strideN) : 0.0f;
#pragma unroll
    for (int r = 0; r < 6; r++) w_bi[r] = in ? __ldg(bi.wn + px_bi + r * strideN) : 0.0f;
    mbar_wait(&sm.bar, 0);

    // ---- slice both lattices separately: the Potts partials, then G_t ----
#ifdef DSRG_NO_TAIL1
    const bool tail1 = false;
#else
    const bool tail1 = (M == MP - 3);
#endif
    float p_sp = 0.0f, p_bi = 0.0f;
    if constexpr (kCompat) {
        if (PH != MODE_FIRST) {
            // S_sp, then S_bi, each sliced into sl (zero outside the image), its mu^T message into G_t and its row
            // parked; Q_t parked beside them
            constexpr int kRow = compat_park_stride(MP);
            const int rs = compat_park_stride(M);
            float *pk_bi = park + tid * rs, *pk_sp = pk_bi + kTileThreads * kRow, *pk_q = pk_sp + kTileThreads * kRow;
            float sl[MP];
#pragma unroll
            for (int k = 0; k < MP; k++) sl[k] = 0.0f;
            if (in) {
                if (!fb_sp)
                    tile_slice_smem<MP, 3>(vs_sp, sp.tl_loc + px_sp, strideN, w_sp, a_sp, sl, tail1);
                else
                    tile_slice_global<MP, 3>(reinterpret_cast<const float4 *>(sp.val_in), sp.off + px_sp, strideN,
                                             base_sp, w_sp, a_sp, sl);
            }
            compat_clear_phantoms<MP>(sl, M);
            compat_apply<MP, true>(mu + MP * MP, sl, t);
#pragma unroll
            for (int k = 0; k < MP; k++) {
                if (k < M) pk_sp[k] = sl[k];
                sl[k] = 0.0f;
            }
            if (in) {
                if (!fb_bi)
                    tile_slice_smem<MP, 6>(vs_bi, bi.tl_loc + px_bi, strideN, w_bi, a_bi, sl, tail1);
                else
                    tile_slice_global<MP, 6>(reinterpret_cast<const float4 *>(bi.val_in), bi.off + px_bi, strideN,
                                             base_bi, w_bi, a_bi, sl);
            }
            compat_clear_phantoms<MP>(sl, M);
            compat_apply<MP, true>(mu, sl, t);
#pragma unroll
            for (int k = 0; k < MP; k++) {
                if (k < M) {
                    pk_bi[k] = sl[k];
                    pk_q[k] = q[k];
                }
            }
        }
    } else if (PH != MODE_FIRST && in) {
        float sl[MP];
#pragma unroll
        for (int k = 0; k < MP; k++) sl[k] = 0.0f;
        if (!fb_sp)
            tile_slice_smem<MP, 3>(vs_sp, sp.tl_loc + px_sp, strideN, w_sp, a_sp, sl, tail1);
        else
            tile_slice_global<MP, 3>(reinterpret_cast<const float4 *>(sp.val_in), sp.off + px_sp, strideN, base_sp,
                                     w_sp, a_sp, sl);
#pragma unroll
        for (int k = 0; k < MP; k++) {
            p_sp = fmaf(sl[k], q[k], p_sp);
            t[k] = w2 * sl[k];
            sl[k] = 0.0f;
        }
        if (!fb_bi)
            tile_slice_smem<MP, 6>(vs_bi, bi.tl_loc + px_bi, strideN, w_bi, a_bi, sl, tail1);
        else
            tile_slice_global<MP, 6>(reinterpret_cast<const float4 *>(bi.val_in), bi.off + px_bi, strideN, base_bi,
                                     w_bi, a_bi, sl);
#pragma unroll
        for (int k = 0; k < MP; k++) {
            p_bi = fmaf(sl[k], q[k], p_bi);
            t[k] = fmaf(w1, sl[k], t[k]);
        }
    }
    // ---- g = Q (G - <G, Q>)  (sumAndNormalize, densecrf.cpp:107-114, with the opposite sign) ----
    float dot = 0.0f;
#pragma unroll
    for (int k = 0; k < MP; k++) dot = fmaf(t[k], q[k], dot);
#pragma unroll
    for (int k = 0; k < MP; k++) t[k] = q[k] * (t[k] - dot);
    if (in) {
        float *gb = gU + ub;
#pragma unroll
        for (int k = 0; k < MP; k++) {
            if (k < M) *gb = (PH == MODE_FIRST) ? t[k] : *gb + t[k];
            gb += N;
        }
    }
    if constexpr ((MODE & MODE_GSTORE) != 0) {   // g_t for the kernel-bandwidth pass of iteration t - 1
        if (in) {
#pragma unroll
            for (int k = 0; k < MP; k++)
                if (k < M) gstore[ub + (size_t)k * N] = t[k];
        }
    }
    // ---- the tile's Potts partials, in a fixed order ----
    if (!kCompat && PH != MODE_FIRST) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            p_sp += __shfl_down_sync(0xffffffffu, p_sp, o);
            p_bi += __shfl_down_sync(0xffffffffu, p_bi, o);
        }
        if ((tid & 31) == 0) red[tid >> 5] = make_float2(p_sp, p_bi);
    }
    if (PH == MODE_LAST) {
        __syncthreads();
    } else {
        // ---- splat g (tile_park's barriers also publish red[]) ----
        const float4 *qs = tile_park(smt, t, w_sp, w_bi);
        float4 *vout_sp = reinterpret_cast<float4 *>(sp.val_out), *vout_bi = reinterpret_cast<float4 *>(bi.val_out);
        if (fb_sp && in) tile_splat_direct<MP, 3>(vout_sp, sp.off + px_sp, strideN, base_sp, w_sp, t);
        if (fb_bi && in) tile_splat_direct<MP, 6>(vout_bi, bi.off + px_bi, strideN, base_bi, w_bi, t);
        tile_splat_csr<MP>(vout_sp, vout_bi, n_sp, n_bi, hdr_sp, hdr_bi, base_sp, base_bi, ent_sp, ent_bi, qs,
                           smt.wtab);
    }
    if constexpr (kCompat) {
        // ---- the tile's two outer-product partials (the barriers above published the parked rows) ----
        float *pp = reinterpret_cast<float *>(part) + ((size_t)b * ntiles + tile) * 2 * M * M;
        const int rs = compat_park_stride(M);
        constexpr int kRow = compat_park_stride(MP);
        const float *pk_bi = park, *pk_sp = park + kTileThreads * kRow, *pk_q = pk_sp + kTileThreads * kRow;
        for (int e = tid; e < M * M; e += kTileThreads) {
            float a_b = 0.0f, a_s = 0.0f;
            if (PH != MODE_FIRST) {
                const int l = e / M, l2 = e - l * M;
                for (int i = 0; i < kTileThreads; i++) {
                    const float qv = pk_q[i * rs + l2];
                    a_b = fmaf(pk_bi[i * rs + l], qv, a_b);
                    a_s = fmaf(pk_sp[i * rs + l], qv, a_s);
                }
                a_b += pp[e];
                a_s += pp[M * M + e];
            }
            pp[e] = a_b;
            pp[M * M + e] = a_s;
        }
    } else if (tid == 0) {
        float2 *pp = part + (size_t)b * ntiles + tile;
        if (PH == MODE_FIRST) {
            *pp = make_float2(0.0f, 0.0f);
        } else {
            float2 a = *pp;
#pragma unroll
            for (int w = 0; w < kTileThreads / 32; w++) {
                a.x += red[w].x;
                a.y += red[w].y;
            }
            *pp = a;
        }
    }
}

// dL/dU = g_0 alone (T = 0: Q_0 = softmax(U))
__global__ void __launch_bounds__(kThreads)
k_mf_softmax_vjp(const float *G, const float *Q, float *gU, int M, int N) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const size_t at = (size_t)b * M * N + i;
    float dot = 0.0f;
    for (int k = 0; k < M; k++) dot = fmaf(G[at + (size_t)k * N], Q[at + (size_t)k * N], dot);
    for (int k = 0; k < M; k++) gU[at + (size_t)k * N] = Q[at + (size_t)k * N] * (G[at + (size_t)k * N] - dot);
}

// per image: the Potts partials of its tiles, summed in a fixed order -> out[b] = {dL/dw1, dL/dw2}
__global__ void __launch_bounds__(kThreads)
k_mf_potts_reduce(const float2 *part, float *out, int ntiles) {
    __shared__ float2 acc[kThreads];
    const int b = blockIdx.x;
    float2 a = make_float2(0.0f, 0.0f);
    for (int i = threadIdx.x; i < ntiles; i += kThreads) {
        const float2 v = part[(size_t)b * ntiles + i];
        a.x += v.x;
        a.y += v.y;
    }
    acc[threadIdx.x] = a;
    __syncthreads();
    for (int o = kThreads / 2; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
            acc[threadIdx.x].x += acc[threadIdx.x + o].x;
            acc[threadIdx.x].y += acc[threadIdx.x + o].y;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        out[2 * b] = acc[0].y;       // bilateral: w1
        out[2 * b + 1] = acc[0].x;   // spatial: w2
    }
}

// per image: the compatibility partials of its tiles, summed in tile order -> out[b] = -sum ([2][M][M], {bi, sp})
__global__ void __launch_bounds__(kThreads)
k_mf_compat_reduce(const float *part, float *out, int ntiles, int mm2) {
    const int b = blockIdx.y;
    const int e = blockIdx.x * kThreads + threadIdx.x;
    if (e >= mm2) return;
    float a = 0.0f;
    for (int i = 0; i < ntiles; i++) a += part[((size_t)b * ntiles + i) * mm2 + e];
    out[(size_t)b * mm2 + e] = -a;
}

// ---------------------------------------------------------------------------------------------
// The kernel-bandwidth gradient (DenseCRF::gradient's kernel_grad under DIAG_KERNEL and NORMALIZE_SYMMETRIC,
// pairwise.cpp:87-97, :175-185).  Per lattice, with x_t = -mu^T g_{t+1}, u_t = -mu Q_t (Potts: w g_{t+1}, w Q_t):
//
//   dL/df = sum_t d^K <n x_t, K (n Q_t)>  -  d^K <c, K 1>,   c = sum_t 1/2 n^3 sum_l (x_t K(n Q_t) + K^T(n x_t) Q_t)
//
// d^K is the derivative through the barycentric weights with simplices, vertices and neighbours held
// (Permutohedral::gradient).  At a pixel's incidence r it needs s_r = n (x . Vy[r] + u . Vg[r]) with
// Vy = B S(n Q_t) (a new splat and forward blur per iteration, k_kg_splatq) and Vg = B^T S(n g_{t+1}), the
// reverse-blurred buffer k_mf_tile_bwd slices at iteration t: mu^T acts label-wise, so B^T S(n x) = -mu^T Vg and
// its dot with n Q is u . Vg.  c at the pixel is 1/2 n^2 alpha sum_r bary_r s_r, so the normalisation term needs
// one splat of the summed c and of ones after the loop (k_kg_splat1, k_kg_norm).  The derivative goes to the
// features through the pixel's ranks (recomputed with the build's arithmetic, simplex.cuh) and the transposed
// elevation matrix, and to the DIAG parameters as dL/dp_i = sum f_i (dL/df)_i.  Each 256-pixel block keeps its seven
// sums in part[b][block] (the first pass writes them), and k_kg_reduce adds the blocks in order: no float atomics.
// ---------------------------------------------------------------------------------------------
// s_r = n * w * (x . Vy[r] + u . Vg[r]) at every incidence of one lattice; c = 1/2 n^2 alpha sum_r bary_r s_r
template <int MP, int D>
__device__ __forceinline__ float kg_incidences(const KgLat &L, int b, int i, int N, const float *x, const float *u,
                                               float w, const float4 *vy, const float4 *vg, float *s) {
    constexpr int CH = MP / 4;
    const size_t at = (size_t)(L.shared ? 0 : b) * (D + 1) * N + i;
    const int base = L.rowbase[b];
    const float n = __ldg(L.norm + (size_t)(L.shared ? 0 : b) * N + i);
    float cs = 0.0f;
#pragma unroll
    for (int r = 0; r <= D; r++) {
        const size_t row = (size_t)(base + __ldg(L.off + at + (size_t)r * N)) * CH;
        float acc = 0.0f;
#pragma unroll
        for (int c = 0; c < CH; c++) {
            const float4 a = vy[row + c], g = vg[row + c];
            acc = fmaf(x[4 * c], a.x, acc);
            acc = fmaf(x[4 * c + 1], a.y, acc);
            acc = fmaf(x[4 * c + 2], a.z, acc);
            acc = fmaf(x[4 * c + 3], a.w, acc);
            acc = fmaf(u[4 * c], g.x, acc);
            acc = fmaf(u[4 * c + 1], g.y, acc);
            acc = fmaf(u[4 * c + 2], g.z, acc);
            acc = fmaf(u[4 * c + 3], g.w, acc);
        }
        s[r] = n * w * acc;
        cs = fmaf(__ldg(L.bary + at + (size_t)r * N), s[r], cs);
    }
    return 0.5f * n * n * L.alpha * cs;
}

// splat wn Q_t into both lattices' zeroed targets (the forward's splat, straight to global rows)
template <int MP>
__global__ void __launch_bounds__(kThreads)
k_kg_splatq(KgArgs a, const float *Qt, float4 *vsp, float4 *vbi) {
    const int b = blockIdx.y, i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= a.N) return;
    float q[MP], w[6];
#pragma unroll
    for (int k = 0; k < MP; k++) q[k] = k < a.M ? __ldg(Qt + ((size_t)b * a.M + k) * a.N + i) : 0.0f;
    const size_t px_sp = (size_t)(a.sp.shared ? 0 : b) * 3 * a.N + i, px_bi = (size_t)(a.bi.shared ? 0 : b) * 6 * a.N + i;
#pragma unroll
    for (int r = 0; r < 3; r++) w[r] = __ldg(a.sp.wn + px_sp + (size_t)r * a.N);
    tile_splat_direct<MP, 3>(vsp, a.sp.off + px_sp, a.N, a.sp.rowbase[b], w, q);
#pragma unroll
    for (int r = 0; r < 6; r++) w[r] = __ldg(a.bi.wn + px_bi + (size_t)r * a.N);
    tile_splat_direct<MP, 6>(vbi, a.bi.off + px_bi, a.N, a.bi.rowbase[b], w, q);
}

// iteration t's lattice terms: g = g_{t+1}, Qt = Q_t, vy_* = B S(n Q_t), vg_* = B^T S(n g_{t+1}); COMPAT: a.potts is
// {mu_bi, mu_sp} ([2][M][M]); FEAT: the bilateral features from feat, their per-pixel dL/df to gfeat (kg_features)
template <int MP, bool COMPAT, bool FEAT>
__device__ __forceinline__ void kg_pass(const KgArgs &a, const float *g, const float *Qt, const float4 *vy_sp,
                                        const float4 *vy_bi, const float4 *vg_sp, const float4 *vg_bi, int first,
                                        const float *feat, float *gfeat) {
    __shared__ float mus[COMPAT ? 2 * MP * MP : 1];
    const int b = blockIdx.y, i = blockIdx.x * kThreads + threadIdx.x;
    const bool in = i < a.N;
    if constexpr (COMPAT) {
        for (int e = threadIdx.x; e < 2 * MP * MP; e += kThreads) {
            const int k = e / (MP * MP), l = e / MP % MP, l2 = e % MP;
            mus[e] = (l < a.M && l2 < a.M) ? __ldg(a.potts + ((size_t)k * a.M + l) * a.M + l2) : 0.0f;
        }
        __syncthreads();
    }
    float dp[7];
#pragma unroll
    for (int k = 0; k < 7; k++) dp[k] = 0.0f;
    if (in) {
        const int x = i % a.W, y = i / a.W;
        float gv[MP], qv[MP];
#pragma unroll
        for (int k = 0; k < MP; k++) {
            gv[k] = k < a.M ? __ldg(g + ((size_t)b * a.M + k) * a.N + i) : 0.0f;
            qv[k] = k < a.M ? __ldg(Qt + ((size_t)b * a.M + k) * a.N + i) : 0.0f;
        }
        float s[6];
        float *csum_sp = a.csum + (size_t)b * a.N + i, *csum_bi = csum_sp + (size_t)gridDim.y * a.N;
        float c_sp, c_bi;
        if constexpr (COMPAT) {
            // x = -mu^T g, u = -mu Q per lattice (mus: {mu_bi, mu_sp})
            float xv[MP], uv[MP];
#pragma unroll
            for (int kk = 0; kk < 2; kk++) {
                const float *mu = mus + (kk == 0 ? MP * MP : 0);
#pragma unroll
                for (int l = 0; l < MP; l++) {
                    float xa = 0.0f, ua = 0.0f;
#pragma unroll
                    for (int l2 = 0; l2 < MP; l2++) {
                        xa = fmaf(-mu[l2 * MP + l], gv[l2], xa);
                        ua = fmaf(-mu[l * MP + l2], qv[l2], ua);
                    }
                    xv[l] = xa;
                    uv[l] = ua;
                }
                if (kk == 0) {
                    c_sp = kg_incidences<MP, 2>(a.sp, b, i, a.N, xv, uv, 1.0f, vy_sp, vg_sp, s);
                    kg_features<2>(a.sp, x, y, a.image, b, a.N, i, s, 1.0f, dp + 5);
                } else {
                    c_bi = kg_incidences<MP, 5>(a.bi, b, i, a.N, xv, uv, 1.0f, vy_bi, vg_bi, s);
                    kg_features<5, FEAT>(a.bi, x, y, a.image, b, a.N, i, s, 1.0f, dp, feat, gfeat, first != 0);
                }
            }
        } else {
            const float w1 = a.potts ? __ldg(a.potts) : a.w1, w2 = a.potts ? __ldg(a.potts + 1) : a.w2;
            c_sp = kg_incidences<MP, 2>(a.sp, b, i, a.N, gv, qv, w2, vy_sp, vg_sp, s);
            kg_features<2>(a.sp, x, y, a.image, b, a.N, i, s, 1.0f, dp + 5);
            c_bi = kg_incidences<MP, 5>(a.bi, b, i, a.N, gv, qv, w1, vy_bi, vg_bi, s);
            kg_features<5, FEAT>(a.bi, x, y, a.image, b, a.N, i, s, 1.0f, dp, feat, gfeat, first != 0);
        }
        *csum_sp = first ? c_sp : *csum_sp + c_sp;
        *csum_bi = first ? c_bi : *csum_bi + c_bi;
    }
    kg_block_sum(a, b, dp, first != 0);
}

template <int MP, bool COMPAT>
__global__ void __launch_bounds__(kThreads)
k_kg_pass(KgArgs a, const float *g, const float *Qt, const float4 *vy_sp, const float4 *vy_bi, const float4 *vg_sp,
          const float4 *vg_bi, int first) {
    kg_pass<MP, COMPAT, false>(a, g, Qt, vy_sp, vy_bi, vg_sp, vg_bi, first, nullptr, nullptr);
}

// k_kg_pass on caller-given bilateral features: feat [B][5][N] in, the pass's dL/df out to gfeat [B][5][N]
template <int MP, bool COMPAT>
__global__ void __launch_bounds__(kThreads)
k_kgf_pass(KgArgs a, const float *g, const float *Qt, const float4 *vy_sp, const float4 *vy_bi, const float4 *vg_sp,
           const float4 *vg_bi, int first, const float *feat, float *gfeat) {
    kg_pass<MP, COMPAT, true>(a, g, Qt, vy_sp, vy_bi, vg_sp, vg_bi, first, feat, gfeat);
}

// the normalisation term's splats, one channel each in 4-wide rows: bary into fw_* (channel 0, blurred in K's order)
// and bary * c into rv_* (channel 1, blurred in K^T's order)
__global__ void __launch_bounds__(kThreads)
k_kg_splat1(KgArgs a, float *fw_sp, float *rv_sp, float *fw_bi, float *rv_bi) {
    const int b = blockIdx.y, i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= a.N) return;
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const KgLat &L = k ? a.bi : a.sp;
        const int dp1 = k ? 6 : 3;
        const float c = a.csum[((size_t)k * gridDim.y + b) * a.N + i];
        const size_t at = (size_t)(L.shared ? 0 : b) * dp1 * a.N + i;
        float *fw = k ? fw_bi : fw_sp, *rv = k ? rv_bi : rv_sp;
        for (int r = 0; r < dp1; r++) {
            const size_t row = (size_t)(L.rowbase[b] + __ldg(L.off + at + (size_t)r * a.N)) * 4;
            const float w = __ldg(L.bary + at + (size_t)r * a.N);
            atomicAdd(fw + row, w);
            atomicAdd(rv + row + 1, w * c);
        }
    }
}

// -d^K <c, K 1> = -(c . B S 1 + 1 . B^T S c) at each incidence, rotated to the features
template <bool FEAT>
__device__ __forceinline__ void kg_norm(const KgArgs &a, const float4 *v1_sp, const float4 *vc_sp,
                                        const float4 *v1_bi, const float4 *vc_bi, const float *feat, float *gfeat) {
    const int b = blockIdx.y, i = blockIdx.x * kThreads + threadIdx.x;
    float dp[7];
#pragma unroll
    for (int k = 0; k < 7; k++) dp[k] = 0.0f;
    if (i < a.N) {
        const int x = i % a.W, y = i / a.W;
        float s[6];
#pragma unroll
        for (int k = 0; k < 2; k++) {
            const KgLat &L = k ? a.bi : a.sp;
            const int dp1 = k ? 6 : 3;
            const float c = a.csum[((size_t)k * gridDim.y + b) * a.N + i];
            const size_t at = (size_t)(L.shared ? 0 : b) * dp1 * a.N + i;
            const float4 *v1 = k ? v1_bi : v1_sp, *vc = k ? vc_bi : vc_sp;
#pragma unroll
            for (int r = 0; r < 6; r++) {
                if (r < dp1) {
                    const size_t row = (size_t)(L.rowbase[b] + __ldg(L.off + at + (size_t)r * a.N));
                    s[r] = fmaf(c, v1[row].x, vc[row].y);
                }
            }
            if (k)
                kg_features<5, FEAT>(L, x, y, a.image, b, a.N, i, s, -1.0f, dp, feat, gfeat, false);
            else
                kg_features<2>(L, x, y, a.image, b, a.N, i, s, -1.0f, dp + 5);
        }
    }
    kg_block_sum(a, b, dp, false);
}

__global__ void __launch_bounds__(kThreads)
k_kg_norm(KgArgs a, const float4 *v1_sp, const float4 *vc_sp, const float4 *v1_bi, const float4 *vc_bi) {
    kg_norm<false>(a, v1_sp, vc_sp, v1_bi, vc_bi, nullptr, nullptr);
}

// k_kg_norm on caller-given bilateral features: adds the normalisation term's dL/df to gfeat
__global__ void __launch_bounds__(kThreads)
k_kgf_norm(KgArgs a, const float4 *v1_sp, const float4 *vc_sp, const float4 *v1_bi, const float4 *vc_bi,
           const float *feat, float *gfeat) {
    kg_norm<true>(a, v1_sp, vc_sp, v1_bi, vc_bi, feat, gfeat);
}

// per image: the blocks' sums in block order -> grad_theta[b] = -dL/dp / theta (theta order)
__global__ void k_kg_reduce(const float *part, int nblk, float *out, KgArgs a) {
    const int b = blockIdx.x, k = threadIdx.x;
    if (k >= 7) return;
    float acc = 0.0f;
    for (int i = 0; i < nblk; i++) acc += part[((size_t)b * nblk + i) * 8 + k];
    const float th = k < 5 ? a.bi.sigma[k] : a.sp.sigma[k - 5];
    out[(size_t)b * 7 + k] = -acc / th;
}

// k_kg_reduce for the spatial bandwidths alone (the feature backward): grad_theta_sp[b] = -dL/dp / theta_gamma
__global__ void k_kgf_reduce_sp(const float *part, int nblk, float *out, KgArgs a) {
    const int b = blockIdx.x, k = threadIdx.x;
    if (k >= 2) return;
    float acc = 0.0f;
    for (int i = 0; i < nblk; i++) acc += part[((size_t)b * nblk + i) * 8 + 5 + k];
    out[(size_t)b * 2 + k] = -acc / a.sp.sigma[k];
}

// the NaN policy of the feature passes (nan_images): every value of a flagged image's slabs becomes NaN
__global__ void __launch_bounds__(kThreads)
k_nan_images(const int *bad, float *p, long long per_image, long long rep_stride) {
    const int b = blockIdx.y, r = blockIdx.z;
    if (!bad[b]) return;
    float *q = p + r * rep_stride + b * per_image;
    for (long long k = blockIdx.x * (long long)kThreads + threadIdx.x; k < per_image; k += (long long)gridDim.x * kThreads)
        q[k] = __int_as_float(0x7fc00000);
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

// tile_major: the forward kernels' view, whose wn / tl_loc are the per-tile blocks (TileLat)
static TileLat make_tile_view(const Lattice &L, const float *val_in, float *val_out, bool tile_major = false) {
    TileLat v;
    v.off = L.off;
    v.rowbase = L.rowbase;
    v.tl_nloc = L.tl_nloc;
    v.tl_hy = L.tl_hy;
    v.tl_hdr = L.tl_hdr;
    v.tl_pack = L.tl_pack;
    v.entcap = L.entcap;
    v.tl_loc = tile_major ? L.tl_li : L.tl_loc;
    v.wn = tile_major ? L.tl_w : L.wn;
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
//
// `reverse` applies the transposed blur K^T of the backward (DenseKernel::filter(..., transpose=true),
// pairwise.cpp:63-80; permutohedral.cpp:556 with reverse: axes d..0): the same passes in the opposite order, each pair
// with its two axes swapped (a negative neighbour stride), so the bilateral lattice runs (5,4) (3,2) (1,0) and the
// spatial one 2 then (1,0).  Each axis' blur is symmetric on the real rows (a missing neighbour is the zero row, which
// stays zero), so K^T is the product of the same axis blurs in the opposite order.
template <int MP>
static float *blur_all(Engine *e, const Lattice &L, float *buf, float *tmp, float *dead, int B, int tag, int grid,
                       cudaStream_t s, bool reverse = false) {
    float *src = buf, *dst = tmp;
    const int npass = L.d / 2 + 1;
    for (int p = 0; p < npass; p++) {
        const int j = 2 * (reverse ? npass - 1 - p : p);  // the pass's lowest axis
        const float4 *in = (const float4 *)src;
        const long long nst = reverse ? -L.nbr_stride : L.nbr_stride;
        const int2 *nbr = L.nbr + (size_t)(reverse && j < L.d ? j + 1 : j) * L.nbr_stride;
        float4 *zero = p == 0 ? (float4 *)dead : nullptr;
        if (j == L.d) {
            DSRG_LAUNCH(e, tag, s, (k_mf_blur<MP, 1, 8><<<grid, kThreads, 0, s>>>(in, (float4 *)dst, nbr, nst,
                                                                                L.rowbase, B, L.shared, zero, 0)));
        } else if (L.shared) {  // the spatial lattice: ~13.5 k rows per image at 321², always cached
            DSRG_LAUNCH(e, tag, s, (k_mf_blur<MP, 2, 4><<<grid, kThreads, 0, s>>>(in, (float4 *)dst, nbr, nst,
                                                                                L.rowbase, B, L.shared, zero, 0)));
        } else if (L.capv <= kBlurCachedRows) {  // no image of this size can have more rows
            DSRG_LAUNCH(e, tag, s, (k_mf_blur<MP, 2, blur_cached_ctas(MP)><<<grid, kThreads, 0, s>>>(
                                       in, (float4 *)dst, nbr, nst, L.rowbase, B, L.shared, zero, 0)));
        } else {
            DSRG_LAUNCH(e, tag, s, (k_mf_blur<MP, 2, blur_cached_ctas(MP)><<<grid, kThreads, 0, s>>>(in, (float4 *)dst, nbr, nst,
                                                                                L.rowbase, B, L.shared, zero, 1)));
            DSRG_LAUNCH(e, tag, s, (k_mf_blur<MP, 2, 4><<<grid, kThreads, 0, s>>>(in, (float4 *)dst, nbr, nst,
                                                                                L.rowbase, B, L.shared, zero, 2)));
        }
        float *t = src;
        src = dst;
        dst = t;
    }
    return src;
}

// q_hist != nullptr: the training forward (MODE_HIST), Q_t of every iteration to q_hist[t] ([T+1][B][M][N]), with
// the Potts weights read from `potts` ({w1, w2}, device) when it is given, or the compatibility matrices `compat`
// ({mu_bi, mu_sp}, device) in their place (MODE_COMPAT).  `compat` without q_hist: the inference with matrices, Q_T
// alone to e->Q0 as the Potts inference leaves it
template <int MP>
static int run_impl(Engine *e, int B, const float *unary, int layout, bool clamp, float *unary_rw,
                    const dsrg_crf_params &p, cudaStream_t s, float *q_hist = nullptr, const float *potts = nullptr,
                    const float *compat = nullptr) {
    const int M = e->M, N = e->N;
    dim3 gp(cdiv(N, kThreads), B);
    const int T = p.n_iters;
    const bool hist = q_hist != nullptr;
    const size_t slab = (size_t)B * M * N;
    // planar (NCHW) callers are read in place by the tile kernel; NHWC callers (and T == 0) go
    // through the layout-converting init kernel
    const bool direct = (layout == DSRG_LAYOUT_NCHW) && T > 0;
    const float *Usrc = direct ? unary : e->U;
    float *Urw = direct ? unary_rw : nullptr;
    const int tclamp = (direct && clamp) ? 1 : 0;
    if (!direct)
        DSRG_LAUNCH(e, T_MF_INIT, s,
                    k_mf_init<MP><<<gp, kThreads, 0, s>>>(unary, unary_rw, layout, clamp ? 1 : 0, e->U,
                                                          T == 0 ? (hist ? q_hist : e->Q0) : nullptr, M, N));
    if (T == 0) return DSRG_OK;
    const float alpha_sp = 1.0f / (1 + powf(2, -e->sp.d));  // permutohedral.cpp:571
    const float alpha_bi = 1.0f / (1 + powf(2, -e->bi.d));
    // device-resident weights: the kernels multiply alpha by them (MODE_HIST)
    const float c_sp = (potts || compat) ? alpha_sp : p.w2 * alpha_sp, c_bi = (potts || compat) ? alpha_bi : p.w1 * alpha_bi;
    float *urw = hist ? const_cast<float *>(potts) : Urw;
    const size_t smem = sizeof(TileSmemFwd<MP>);
    const size_t smem_hy = sizeof(TileSmemFwd<MP, kMaxLocHy>);
    const size_t smem_c = smem + kCompatSmem<MP>, smem_hy_c = smem_hy + kCompatSmem<MP>;
    static bool attr_done[64] = {false};   // function attributes are per device
    const int dv = e->device & 63;
    if (!attr_done[dv]) {
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_FIRST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_MID>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_LAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_FIRST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_MID>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_LAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_FIRST | MODE_HIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_MID | MODE_HIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_LAST | MODE_HIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_FIRST | MODE_HIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_MID | MODE_HIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_LAST | MODE_HIST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_MID | MODE_HIST | MODE_COMPAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_LAST | MODE_HIST | MODE_COMPAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_MID | MODE_HIST | MODE_COMPAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy_c));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_LAST | MODE_HIST | MODE_COMPAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy_c));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_MID | MODE_COMPAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile<MP, MODE_LAST | MODE_COMPAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_MID | MODE_COMPAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy_c));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_hy<MP, MODE_LAST | MODE_COMPAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_hy_c));
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
#define DSRG_TILE_LAUNCH_AT(MODEV, QOUT, URW, SMEM, SMEM_HY)                                                          \
    do {                                                                                                              \
        if (hy_on)                                                                                                    \
            DSRG_LAUNCH(e, T_MF_TILE_HY, s,                                                                           \
                        (k_mf_tile_hy<MP, MODEV><<<hgrid, kTileThreads, SMEM_HY, s>>>(                                \
                            Usrc, URW, tclamp, QOUT, vsp, vbi, c_sp, c_bi, M, N, e->W, e->H, e->tiles_x, e->ntiles,   \
                            e->tile_w, e->hy_list, e->hy_count)));                                                    \
        DSRG_LAUNCH(e, T_MF_TILE, s,                                                                                  \
                    (k_mf_tile<MP, MODEV><<<gt, kTileThreads, SMEM, s>>>(Usrc, URW, tclamp, QOUT, vsp, vbi, c_sp,     \
                                                                        c_bi, M, N, e->W, e->H, e->tiles_x,           \
                                                                        e->ntiles, e->tile_w)));                      \
    } while (0)
#define DSRG_TILE_LAUNCH(MODEV, QOUT) DSRG_TILE_LAUNCH_AT(MODEV, QOUT, urw, smem, smem_hy)
#define DSRG_TILE_LAUNCH_COMPAT(MODEV, QOUT)                                                                          \
    DSRG_TILE_LAUNCH_AT(MODEV | MODE_HIST | MODE_COMPAT, QOUT, const_cast<float *>(compat), smem_c, smem_hy_c)
    for (int it = 0; it <= T; it++) {
        TileLat vsp = make_tile_view(e->sp, spX, spY, true), vbi = make_tile_view(e->bi, biX, biY, true);
        if (compat && !hist) {
            // the matrices passed as the matrices, never as the clamp's U_rw; the first iteration is the Potts one
            if (it == T) {
                DSRG_TILE_LAUNCH_AT(MODE_LAST | MODE_COMPAT, e->Q0, const_cast<float *>(compat), smem_c, smem_hy_c);
                break;
            }
            if (it == 0)
                DSRG_TILE_LAUNCH_AT(MODE_FIRST, nullptr, nullptr, smem, smem_hy);
            else
                DSRG_TILE_LAUNCH_AT(MODE_MID | MODE_COMPAT, nullptr, const_cast<float *>(compat), smem_c, smem_hy_c);
        } else if (compat) {
            // the first iteration slices nothing: the plain training kernel, without weights
            float *qt = q_hist + (size_t)it * slab;
            if (it == T) {
                DSRG_TILE_LAUNCH_COMPAT(MODE_LAST, qt);
                break;
            }
            if (it == 0)
                DSRG_TILE_LAUNCH_AT(MODE_FIRST | MODE_HIST, qt, nullptr, smem, smem_hy);
            else
                DSRG_TILE_LAUNCH_COMPAT(MODE_MID, qt);
        } else if (hist) {
            float *qt = q_hist + (size_t)it * slab;
            if (it == T) {
                DSRG_TILE_LAUNCH(MODE_LAST | MODE_HIST, qt);
                break;
            }
            if (it == 0)
                DSRG_TILE_LAUNCH(MODE_FIRST | MODE_HIST, qt);
            else
                DSRG_TILE_LAUNCH(MODE_MID | MODE_HIST, qt);
        } else {
            if (it == T) {
                DSRG_TILE_LAUNCH(MODE_LAST, e->Q0);
                break;
            }
            if (it == 0)
                DSRG_TILE_LAUNCH(MODE_FIRST, nullptr);
            else
                DSRG_TILE_LAUNCH(MODE_MID, nullptr);
        }
        // the old X is dead: the first blur pass clears it and it becomes the next splat target
        float *sp_res = blur_all<MP>(e, e->sp, spY, spZ, spX, B, T_MF_BLUR_SP, bgrid, s);
        float *bi_res = blur_all<MP>(e, e->bi, biY, biZ, biX, B, T_MF_BLUR_BI, bgrid, s);
        float *sp_other = (sp_res == spY) ? spZ : spY, *bi_other = (bi_res == biY) ? biZ : biY;
        float *nspY = spX, *nbiY = biX;
        spX = sp_res; spY = nspY; spZ = sp_other;
        biX = bi_res; biY = nbiY; biZ = bi_other;
    }
#undef DSRG_TILE_LAUNCH_COMPAT
#undef DSRG_TILE_LAUNCH
#undef DSRG_TILE_LAUNCH_AT
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

// The backward of a training forward (DenseCRF::gradient, densecrf.cpp:238-297) on the lattices the pass just built:
// k_mf_tile_bwd from T down to 0 with the transposed blur in between, then the per-image Potts sums -- or, with
// `compat` ({mu_bi, mu_sp}), the MODE_COMPAT kernels and the per-image compatibility sums to g_compat ([B][2][M][M]).
KgLat kg_lat(const Lattice &L) {
    KgLat k;
    k.off = L.off;
    k.bary = L.bary;
    k.wn = L.wn;
    k.norm = L.norm;
    k.rowbase = L.rowbase;
    k.shared = L.shared;
    k.alpha = 1.0f / (1 + powf(2, -L.d));
    for (int i = 0; i < 5; i++) {
        k.sigma[i] = L.sigma[i];
        k.scale[i] = L.scale[i];
    }
    return k;
}

// Iteration t's kernel-bandwidth terms (before k_mf_tile_bwd of iteration t overwrites e->kg_g = g_{t+1}): splat
// n Q_t, blur it in K's order into the kernel-gradient buffers, and k_kg_pass against spX / biX = B^T S(n g_{t+1}).
// With caller-given bilateral features (`feat`) k_kgf_pass, which also writes (first) or adds the per-pixel dL/df to
// gfeat; every launch is timed under `tag`.
template <int MP>
static void kg_iter(Engine *e, const KgArgs &ka, bool compat, int B, const float *qt, const float *spX,
                    const float *biX, bool first, int bgrid, cudaStream_t s, const float *feat, float *gfeat, int tag) {
    const dim3 gp(ka.nblk, B);
    DSRG_LAUNCH(e, tag, s,
                k_mf_zero<MP><<<bgrid, kThreads, 0, s>>>((float4 *)e->kg_sp[0], e->sp.rowbase, (float4 *)e->kg_bi[0],
                                                         e->bi.rowbase, B));
    DSRG_LAUNCH(e, tag, s,
                k_kg_splatq<MP><<<gp, kThreads, 0, s>>>(ka, qt, (float4 *)e->kg_sp[0], (float4 *)e->kg_bi[0]));
    const float *vy_sp = blur_all<MP>(e, e->sp, e->kg_sp[0], e->kg_sp[1], nullptr, B, tag, bgrid, s);
    const float *vy_bi = blur_all<MP>(e, e->bi, e->kg_bi[0], e->kg_bi[1], nullptr, B, tag, bgrid, s);
    if (feat) {
        if (compat)
            DSRG_LAUNCH(e, tag, s,
                        (k_kgf_pass<MP, true><<<gp, kThreads, 0, s>>>(ka, e->kg_g, qt, (const float4 *)vy_sp,
                                                                     (const float4 *)vy_bi, (const float4 *)spX,
                                                                     (const float4 *)biX, first, feat, gfeat)));
        else
            DSRG_LAUNCH(e, tag, s,
                        (k_kgf_pass<MP, false><<<gp, kThreads, 0, s>>>(ka, e->kg_g, qt, (const float4 *)vy_sp,
                                                                      (const float4 *)vy_bi, (const float4 *)spX,
                                                                      (const float4 *)biX, first, feat, gfeat)));
        return;
    }
    if (compat)
        DSRG_LAUNCH(e, T_KGRAD, s,
                    (k_kg_pass<MP, true><<<gp, kThreads, 0, s>>>(ka, e->kg_g, qt, (const float4 *)vy_sp,
                                                                (const float4 *)vy_bi, (const float4 *)spX,
                                                                (const float4 *)biX, first)));
    else
        DSRG_LAUNCH(e, T_KGRAD, s,
                    (k_kg_pass<MP, false><<<gp, kThreads, 0, s>>>(ka, e->kg_g, qt, (const float4 *)vy_sp,
                                                                 (const float4 *)vy_bi, (const float4 *)spX,
                                                                 (const float4 *)biX, first)));
}

// (every launch of the kernel-bandwidth passes is timed under T_KGRAD, of the feature passes under T_FGRAD)
// After the loop: the normalisation term from the summed c, then the per-image sums.  The mean-field buffers are free
// by now: spA / biA take the reverse-blurred splat of c, the kernel-gradient buffers the forward-blurred one of ones.
// With `feat`: k_kgf_norm adds the term's dL/df to gfeat, and only the spatial sums are reduced (to g_theta [B][2],
// when given).
void kg_finish(Engine *e, const KgArgs &ka, int B, float *g_theta, int bgrid, cudaStream_t s, const float *feat,
               float *gfeat, int tag) {
    const dim3 gp(ka.nblk, B);
    DSRG_LAUNCH(e, tag, s,
                k_mf_zero<4><<<bgrid, kThreads, 0, s>>>((float4 *)e->kg_sp[0], e->sp.rowbase, (float4 *)e->kg_bi[0],
                                                        e->bi.rowbase, B));
    DSRG_LAUNCH(e, tag, s,
                k_mf_zero<4><<<bgrid, kThreads, 0, s>>>((float4 *)e->spA, e->sp.rowbase, (float4 *)e->biA,
                                                        e->bi.rowbase, B));
    DSRG_LAUNCH(e, tag, s, k_kg_splat1<<<gp, kThreads, 0, s>>>(ka, e->kg_sp[0], e->spA, e->kg_bi[0], e->biA));
    const float *v1_sp = blur_all<4>(e, e->sp, e->kg_sp[0], e->kg_sp[1], nullptr, B, tag, bgrid, s);
    const float *v1_bi = blur_all<4>(e, e->bi, e->kg_bi[0], e->kg_bi[1], nullptr, B, tag, bgrid, s);
    const float *vc_sp = blur_all<4>(e, e->sp, e->spA, e->spB, nullptr, B, tag, bgrid, s, true);
    const float *vc_bi = blur_all<4>(e, e->bi, e->biA, e->biB, nullptr, B, tag, bgrid, s, true);
    if (feat) {
        DSRG_LAUNCH(e, tag, s,
                    k_kgf_norm<<<gp, kThreads, 0, s>>>(ka, (const float4 *)v1_sp, (const float4 *)vc_sp,
                                                       (const float4 *)v1_bi, (const float4 *)vc_bi, feat, gfeat));
        if (g_theta) DSRG_LAUNCH(e, tag, s, k_kgf_reduce_sp<<<B, 32, 0, s>>>(ka.part, ka.nblk, g_theta, ka));
        return;
    }
    DSRG_LAUNCH(e, tag, s,
                k_kg_norm<<<gp, kThreads, 0, s>>>(ka, (const float4 *)v1_sp, (const float4 *)vc_sp,
                                                  (const float4 *)v1_bi, (const float4 *)vc_bi));
    DSRG_LAUNCH(e, tag, s, k_kg_reduce<<<B, 32, 0, s>>>(ka.part, ka.nblk, g_theta, ka));
}

template <int MP>
static int bwd_impl(Engine *e, int B, const CrfTrainIo &io, const dsrg_crf_params &p, cudaStream_t s) {
    const int M = e->M, N = e->N, T = p.n_iters;
    const size_t slab = (size_t)B * M * N;
    const float *compat = io.compat, *feat = io.features;
    float *g_feat = io.grad_features;
    if (T == 0) {
        if (g_feat) DSRG_CUDA_TRY(cudaMemsetAsync(g_feat, 0, sizeof(float) * 5 * N * B, s));
        if (io.grad_theta_sp) DSRG_CUDA_TRY(cudaMemsetAsync(io.grad_theta_sp, 0, sizeof(float) * 2 * B, s));
        DSRG_LAUNCH(e, T_MF_INIT, s,
                    k_mf_softmax_vjp<<<dim3(cdiv(N, kThreads), B), kThreads, 0, s>>>(io.grad_q, io.q_hist,
                                                                                      io.grad_unary, M, N));
        if (io.grad_potts) DSRG_CUDA_TRY(cudaMemsetAsync(io.grad_potts, 0, sizeof(float) * 2 * B, s));
        if (io.grad_compat) DSRG_CUDA_TRY(cudaMemsetAsync(io.grad_compat, 0, sizeof(float) * 2 * M * M * B, s));
        if (io.grad_theta) DSRG_CUDA_TRY(cudaMemsetAsync(io.grad_theta, 0, sizeof(float) * 7 * B, s));
        DSRG_CUDA_TRY(cudaGetLastError());
        return DSRG_OK;
    }
    static bool attr_done[64] = {false};
    const int dv = e->device & 63;
    const size_t smem = sizeof(TileSmem<MP>);
    const size_t smem_c = smem + kCompatSmem<MP> + kCompatParkSmem<MP>;
    if (!attr_done[dv]) {
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_bwd<MP, MODE_FIRST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_bwd<MP, MODE_MID>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_bwd<MP, MODE_LAST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_bwd<MP, MODE_FIRST | MODE_COMPAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_bwd<MP, MODE_MID | MODE_COMPAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_bwd<MP, MODE_LAST | MODE_COMPAT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_bwd<MP, MODE_FIRST | MODE_GSTORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_bwd<MP, MODE_MID | MODE_GSTORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_bwd<MP, MODE_FIRST | MODE_COMPAT | MODE_GSTORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
        DSRG_CUDA_TRY(cudaFuncSetAttribute(k_mf_tile_bwd<MP, MODE_MID | MODE_COMPAT | MODE_GSTORE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_c));
        attr_done[dv] = true;
    }
    const float a_sp = 1.0f / (1 + powf(2, -e->sp.d)), a_bi = 1.0f / (1 + powf(2, -e->bi.d));
    const int bgrid = DSRG_BLUR_GRID * e->sm_count;
    const dim3 gt(e->ntiles, B);
    float *spX = e->spA, *spY = e->spB, *spZ = e->spC;
    float *biX = e->biA, *biY = e->biB, *biZ = e->biC;
    DSRG_LAUNCH(e, T_MF_ZERO, s,
                k_mf_zero<MP><<<bgrid, kThreads, 0, s>>>((float4 *)spY, e->sp.rowbase, (float4 *)biY, e->bi.rowbase, B));
    // the kernel-bandwidth gradient (g_theta): g_t stored by the launches (MODE_GSTORE), k_kg_pass per iteration;
    // the feature gradient (g_feat) runs the same flow on the kgf kernels and keeps grad_theta_sp for the spatial sums
    float *g_theta = g_feat ? io.grad_theta_sp : io.grad_theta;
    const bool kg = g_theta || g_feat;
    const int kg_tag = g_feat ? T_FGRAD : T_KGRAD;
    KgArgs ka{};
    if (kg) {
        ka.sp = kg_lat(e->sp);
        ka.bi = kg_lat(e->bi);
        ka.image = io.image;
        ka.potts = compat ? compat : io.potts;
        ka.w1 = p.w1;
        ka.w2 = p.w2;
        ka.part = e->kg_part;
        ka.csum = e->kg_csum;
        ka.M = M;
        ka.N = N;
        ka.W = e->W;
        ka.nblk = cdiv(N, kThreads);
    }
#define DSRG_BWD_LAUNCH_AT(MODEV, WP, PART, SMEM)                                                                     \
    DSRG_LAUNCH(e, T_MF_TILE, s,                                                                                      \
                (k_mf_tile_bwd<MP, MODEV><<<gt, kTileThreads, SMEM, s>>>(io.grad_q, qt, io.grad_unary, vsp, vbi, a_sp, \
                                                                        a_bi, WP, p.w1, p.w2, PART, M, N, e->W, e->H, \
                                                                        e->tiles_x, e->ntiles, e->tile_w,             \
                                                                        ((MODEV) & MODE_GSTORE) ? e->kg_g : nullptr)))
#define DSRG_BWD_LAUNCH(MODEV) DSRG_BWD_LAUNCH_AT(MODEV, io.potts, e->potts_part, smem)
#define DSRG_BWD_LAUNCH_COMPAT(MODEV)                                                                                 \
    DSRG_BWD_LAUNCH_AT(MODEV | MODE_COMPAT, compat, reinterpret_cast<float2 *>(e->compat_part), smem_c)
    for (int it = T; it >= 0; it--) {
        const TileLat vsp = make_tile_view(e->sp, spX, spY), vbi = make_tile_view(e->bi, biX, biY);
        const float *qt = io.q_hist + (size_t)it * slab;
        if (kg && it < T)
            kg_iter<MP>(e, ka, compat != nullptr, B, qt, spX, biX, it == T - 1, bgrid, s, feat, g_feat, kg_tag);
        if (compat) {
            if (it == 0) {
                DSRG_BWD_LAUNCH_COMPAT(MODE_LAST);
                break;
            }
            if (kg) {
                if (it == T)
                    DSRG_BWD_LAUNCH_COMPAT(MODE_FIRST | MODE_GSTORE);
                else
                    DSRG_BWD_LAUNCH_COMPAT(MODE_MID | MODE_GSTORE);
            } else if (it == T) {
                DSRG_BWD_LAUNCH_COMPAT(MODE_FIRST);
            } else {
                DSRG_BWD_LAUNCH_COMPAT(MODE_MID);
            }
        } else if (it == 0) {
            DSRG_BWD_LAUNCH(MODE_LAST);
            break;
        } else if (kg) {
            if (it == T)
                DSRG_BWD_LAUNCH(MODE_FIRST | MODE_GSTORE);
            else
                DSRG_BWD_LAUNCH(MODE_MID | MODE_GSTORE);
        } else if (it == T) {
            DSRG_BWD_LAUNCH(MODE_FIRST);
        } else {
            DSRG_BWD_LAUNCH(MODE_MID);
        }
        float *sp_res = blur_all<MP>(e, e->sp, spY, spZ, spX, B, T_MF_BLUR_SP, bgrid, s, true);
        float *bi_res = blur_all<MP>(e, e->bi, biY, biZ, biX, B, T_MF_BLUR_BI, bgrid, s, true);
        float *sp_other = (sp_res == spY) ? spZ : spY, *bi_other = (bi_res == biY) ? biZ : biY;
        float *nspY = spX, *nbiY = biX;
        spX = sp_res; spY = nspY; spZ = sp_other;
        biX = bi_res; biY = nbiY; biZ = bi_other;
    }
#undef DSRG_BWD_LAUNCH_COMPAT
#undef DSRG_BWD_LAUNCH
#undef DSRG_BWD_LAUNCH_AT
    if (io.grad_compat) compat_reduce(e, e->compat_part, io.grad_compat, e->ntiles, 2 * M * M, B, T_MF_EXPORT, s);
    if (io.grad_potts) potts_reduce(e, e->potts_part, io.grad_potts, e->ntiles, B, T_MF_EXPORT, s);
    if (kg) kg_finish(e, ka, B, g_theta, bgrid, s, feat, g_feat, kg_tag);
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int meanfield_run_train(Engine *e, int B, const CrfTrainIo &io, const dsrg_crf_params &p, cudaStream_t s) {
    switch (e->MP) {
#define DSRG_CASE(MPV) \
    case MPV:          \
        return run_impl<MPV>(e, B, io.unary, DSRG_LAYOUT_NCHW, false, nullptr, p, s, io.q_out, io.potts, io.compat);
        DSRG_CASE(4) DSRG_CASE(8) DSRG_CASE(12) DSRG_CASE(16) DSRG_CASE(20) DSRG_CASE(24) DSRG_CASE(28) DSRG_CASE(32)
#undef DSRG_CASE
    }
    set_error("unsupported label count %d", e->M);
    return DSRG_E_INVALID;
}

int meanfield_backward(Engine *e, int B, const CrfTrainIo &io, const dsrg_crf_params &p, cudaStream_t s) {
    switch (e->MP) {
#define DSRG_CASE(MPV) \
    case MPV: return bwd_impl<MPV>(e, B, io, p, s);
        DSRG_CASE(4) DSRG_CASE(8) DSRG_CASE(12) DSRG_CASE(16) DSRG_CASE(20) DSRG_CASE(24) DSRG_CASE(28) DSRG_CASE(32)
#undef DSRG_CASE
    }
    set_error("unsupported label count %d", e->M);
    return DSRG_E_INVALID;
}

void nan_images(Engine *e, const int *bad, float *p, int B, long long per_image, int reps, cudaStream_t s, int tag) {
    const int nblk = cdiv(per_image, kThreads);
    const dim3 gp(nblk < 64 ? nblk : 64, B, reps);
    DSRG_LAUNCH(e, tag, s, k_nan_images<<<gp, kThreads, 0, s>>>(bad, p, per_image, B * per_image));
}

void potts_reduce(Engine *e, const float2 *part, float *out, int nparts, int B, int tag, cudaStream_t s) {
    DSRG_LAUNCH(e, tag, s, k_mf_potts_reduce<<<B, kThreads, 0, s>>>(part, out, nparts));
}

void compat_reduce(Engine *e, const float *part, float *out, int nparts, int mm2, int B, int tag, cudaStream_t s) {
    DSRG_LAUNCH(e, tag, s,
                k_mf_compat_reduce<<<dim3(cdiv(mm2, kThreads), B), kThreads, 0, s>>>(part, out, nparts, mm2));
}

int meanfield_run(Engine *e, int B, const float *unary, int unary_layout, bool clamp_inplace,
                  float *unary_rw, const dsrg_crf_params &p, cudaStream_t s, const float *compat) {
    if (e->MP > DSRG_MAX_LABELS)
        return meanfield_run_wide(e, B, unary, unary_layout, clamp_inplace, unary_rw, p, s, compat);
    switch (e->MP) {
#define DSRG_CASE(MPV) \
    case MPV: return run_impl<MPV>(e, B, unary, unary_layout, clamp_inplace, unary_rw, p, s, nullptr, nullptr, compat);
        DSRG_CASE(4) DSRG_CASE(8) DSRG_CASE(12) DSRG_CASE(16) DSRG_CASE(20) DSRG_CASE(24) DSRG_CASE(28) DSRG_CASE(32)
#undef DSRG_CASE
    }
    set_error("unsupported label count %d", e->M);
    return DSRG_E_INVALID;
}

int meanfield_export(Engine *e, int B, float *out, int layout, cudaStream_t s) {
    dim3 gp(cdiv(e->N, kThreads), B);
    DSRG_LAUNCH(e, T_MF_EXPORT, s, k_mf_export<<<gp, kThreads, 0, s>>>(e->Q0, out, layout, e->M, e->N));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int meanfield_export_map(Engine *e, int B, int32_t *labels, cudaStream_t s) {
    dim3 gp(cdiv(e->N, kThreads), B);
    DSRG_LAUNCH(e, T_MF_EXPORT, s, k_mf_export_map<<<gp, kThreads, 0, s>>>(e->Q0, labels, e->M, e->N));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int meanfield_export_renorm(Engine *e, int B, float *result_out, float *log_out, cudaStream_t s) {
    dim3 gp(cdiv(e->N, kThreads), B);
    DSRG_LAUNCH(e, T_MF_EXPORT, s, k_mf_export_renorm<<<gp, kThreads, 0, s>>>(e->Q0, result_out, log_out, e->M, e->N));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

// ---------------------------------------------------------------------------------------------
// The energy of given marginals (DenseCRF::klDivergence, densecrf.cpp:213-235) and its gradient to them.  Per lattice
// F(Q) = n K(n Q), the message the mean field subtracts (t = unary - mu_sp F_sp(Q) - mu_bi F_bi(Q), Potts mu = -w I):
//   terms[b] = {sum Q log max(Q, 1e-20), -sum unary Q, sum Q . mu_sp F_sp(Q), sum Q . mu_bi F_bi(Q)}
// k_kg_splatq splats wn Q (wn = bary n) into each lattice and blur_all blurs it in K's order; the gradient blurs a
// copy of the splat in K^T's order too, since the device's K is not symmetric (DESIGN.md section 1):
//   grad_q = g0 (Q > 1e-20 ? log Q + 1 : log 1e-20) - g1 unary + sum_k g_k (mu_k F_k(Q) + mu_k^T F_k^T(Q))
// k_crf_energy slices both per pixel as the tile kernels do (weights alpha wn, an fma chain from zero).  The forward's
// per-pixel terms go to per-block double sums part [B][nblk][4], which k_crf_energy_reduce adds in block order: no
// float atomics in the sums, only in the splats.
// ---------------------------------------------------------------------------------------------
struct EnergyArgs {
    KgLat sp, bi;
    const float *q, *unary;     // [B][M][N]; unary may be nullptr (no unary term)
    const float *potts;         // {w1, w2} on the device, or nullptr: w1, w2
    const float *compat;        // {mu_bi, mu_sp} [2][M][M], or nullptr: Potts
    float w1, w2;
    const float *grad_terms;    // [B][4] (the backward)
    float *grad_q, *grad_unary; // [B][M][N]; grad_unary may be nullptr
    double *part;               // [B][nblk][4] (the forward)
    int M, N, nblk;
};

// F(Q) of one lattice at pixel i from its blurred values v: alpha sum_r wn_r v[row_r]
template <int MP, int D>
__device__ __forceinline__ void energy_slice(const KgLat &L, int b, int i, int N, const float4 *v, float *f) {
    constexpr int CH = MP / 4;
    const size_t at = (size_t)(L.shared ? 0 : b) * (D + 1) * N + i;
    const int base = L.rowbase[b];
#pragma unroll
    for (int k = 0; k < MP; k++) f[k] = 0.0f;
#pragma unroll
    for (int r = 0; r <= D; r++) {
        const float w = L.alpha * __ldg(L.wn + at + (size_t)r * N);
        const size_t row = (size_t)(base + __ldg(L.off + at + (size_t)r * N)) * CH;
#pragma unroll
        for (int c = 0; c < CH; c++) {
            const float4 a = v[row + c];
            f[4 * c] = fmaf(w, a.x, f[4 * c]);
            f[4 * c + 1] = fmaf(w, a.y, f[4 * c + 1]);
            f[4 * c + 2] = fmaf(w, a.z, f[4 * c + 2]);
            f[4 * c + 3] = fmaf(w, a.w, f[4 * c + 3]);
        }
    }
}

// message l of lattice kk (0 spatial, 1 bilateral): (mu f)_l, Potts -w f_l
template <int MP, bool COMPAT>
__device__ __forceinline__ float energy_msg(const float *mus, int kk, float w, const float *f, int l) {
    if constexpr (COMPAT) {
        const float *mu = mus + (kk == 0 ? MP * MP : 0);   // mus: {mu_bi, mu_sp}
        float m = 0.0f;
#pragma unroll
        for (int l2 = 0; l2 < MP; l2++) m = fmaf(mu[l * MP + l2], f[l2], m);
        return m;
    } else {
        return -w * f[l];
    }
}

// one pixel per thread: vf_* = K S(wn Q), with BWD vt_* = K^T S(wn Q) too
template <int MP, bool COMPAT, bool BWD>
__global__ void __launch_bounds__(kThreads)
k_crf_energy(EnergyArgs a, const float4 *vf_sp, const float4 *vf_bi, const float4 *vt_sp, const float4 *vt_bi) {
    __shared__ float mus[COMPAT ? 2 * MP * MP : 1];
    __shared__ double red[kThreads / 32][4];
    const int b = blockIdx.y, i = blockIdx.x * kThreads + threadIdx.x;
    if constexpr (COMPAT) {
        for (int e = threadIdx.x; e < 2 * MP * MP; e += kThreads) {
            const int k = e / (MP * MP), l = e / MP % MP, l2 = e % MP;
            mus[e] = (l < a.M && l2 < a.M) ? __ldg(a.compat + ((size_t)k * a.M + l) * a.M + l2) : 0.0f;
        }
        __syncthreads();
    }
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (i < a.N) {
        const float w1 = a.potts ? __ldg(a.potts) : a.w1, w2 = a.potts ? __ldg(a.potts + 1) : a.w2;
        float g0 = 0.0f, g1 = 0.0f, g2 = 0.0f, g3 = 0.0f;
        if constexpr (BWD) {
            g0 = __ldg(a.grad_terms + 4 * b);
            g1 = __ldg(a.grad_terms + 4 * b + 1);
            g2 = __ldg(a.grad_terms + 4 * b + 2);
            g3 = __ldg(a.grad_terms + 4 * b + 3);
        }
        float q[MP], f[MP], g[MP];
#pragma unroll
        for (int k = 0; k < MP; k++) {
            q[k] = 0.0f;
            g[k] = 0.0f;
            if (k < a.M) {
                const size_t at = ((size_t)b * a.M + k) * a.N + i;
                q[k] = __ldg(a.q + at);
                const float u = a.unary ? __ldg(a.unary + at) : 0.0f;
                const float lq = logf(fmaxf(q[k], 1e-20f));
                acc[0] = fmaf(q[k], lq, acc[0]);
                acc[1] = fmaf(-u, q[k], acc[1]);
                if constexpr (BWD) {
                    g[k] = fmaf(-g1, u, g0 * (q[k] > 1e-20f ? lq + 1.0f : lq));
                    if (a.grad_unary) a.grad_unary[at] = -g1 * q[k];
                }
            }
        }
        // one lattice at a time (not unrolled: two copies of the M x M products would not fit the registers)
#pragma unroll 1
        for (int kk = 0; kk < 2; kk++) {
            const float w = kk == 0 ? w2 : w1, gk = kk == 0 ? g2 : g3;
            if (kk == 0)
                energy_slice<MP, 2>(a.sp, b, i, a.N, vf_sp, f);
            else
                energy_slice<MP, 5>(a.bi, b, i, a.N, vf_bi, f);
            float ek = 0.0f;
#pragma unroll
            for (int l = 0; l < MP; l++) {
                const float m = energy_msg<MP, COMPAT>(mus, kk, w, f, l);
                ek = fmaf(q[l], m, ek);
                if constexpr (BWD) g[l] = fmaf(gk, m, g[l]);
            }
            if (kk == 0)
                acc[2] = ek;
            else
                acc[3] = ek;
            if constexpr (BWD) {
                if (kk == 0)
                    energy_slice<MP, 2>(a.sp, b, i, a.N, vt_sp, f);
                else
                    energy_slice<MP, 5>(a.bi, b, i, a.N, vt_bi, f);
                if constexpr (COMPAT) {
                    // g += g_k mu^T f, as mu's rows l2 scaled by g_k f[l2]
                    const float *mu = mus + (kk == 0 ? MP * MP : 0);
#pragma unroll
                    for (int l2 = 0; l2 < MP; l2++) {
                        const float c = gk * f[l2];
#pragma unroll
                        for (int l = 0; l < MP; l++) g[l] = fmaf(mu[l2 * MP + l], c, g[l]);
                    }
                } else {
#pragma unroll
                    for (int l = 0; l < MP; l++) g[l] = fmaf(gk, -w * f[l], g[l]);
                }
            }
        }
        if constexpr (BWD) {
#pragma unroll
            for (int k = 0; k < MP; k++)
                if (k < a.M) a.grad_q[((size_t)b * a.M + k) * a.N + i] = g[k];
        }
    }
    if constexpr (!BWD) {
        double v[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            v[k] = acc[k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], o);
        }
        if ((threadIdx.x & 31) == 0) {
#pragma unroll
            for (int k = 0; k < 4; k++) red[threadIdx.x >> 5][k] = v[k];
        }
        __syncthreads();
        if (threadIdx.x < 4) {
            double s = 0.0;
            for (int w = 0; w < kThreads / 32; w++) s += red[w][threadIdx.x];
            a.part[((size_t)b * a.nblk + blockIdx.x) * 4 + threadIdx.x] = s;
        }
    }
}

// copy the B images' rows of both lattices' splat targets (row counts device-resident, as k_mf_zero)
template <int MP>
__global__ void __launch_bounds__(kThreads)
k_crf_energy_copy(const float4 *a, float4 *a2, const int32_t *rowbase_a, const float4 *c, float4 *c2,
                  const int32_t *rowbase_c, int B) {
    constexpr int CH = MP / 4;
    const long long na = (long long)rowbase_a[B] * CH, nc = (long long)rowbase_c[B] * CH;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < na + nc;
         t += (long long)gridDim.x * blockDim.x) {
        if (t < na) a2[t] = a[t]; else c2[t - na] = c[t - na];
    }
}

// per image: the blocks' sums in block order -> terms[b][4]
__global__ void k_crf_energy_reduce(const double *part, int nblk, float *terms) {
    const int b = blockIdx.x, k = threadIdx.x;
    if (k >= 4) return;
    double s = 0.0;
    for (int i = 0; i < nblk; i++) s += part[((size_t)b * nblk + i) * 4 + k];
    terms[(size_t)b * 4 + k] = (float)s;
}

template <int MP>
static int energy_impl(Engine *e, int B, const float *q, const float *unary, const float *potts, const float *compat,
                       const dsrg_crf_params &p, float *terms, const float *grad_terms, float *grad_q,
                       float *grad_unary, cudaStream_t s) {
    const bool bwd = grad_terms != nullptr;
    KgArgs ka{};
    ka.sp = kg_lat(e->sp);
    ka.bi = kg_lat(e->bi);
    ka.M = e->M;
    ka.N = e->N;
    ka.W = e->W;
    ka.nblk = cdiv(e->N, kThreads);
    EnergyArgs ea{ka.sp, ka.bi, q, unary, potts, compat, p.w1, p.w2, grad_terms, grad_q, grad_unary, e->en_part,
                  e->M, e->N, ka.nblk};
    const int bgrid = DSRG_BLUR_GRID * e->sm_count;
    const dim3 gp(ka.nblk, B);
    // S(wn Q) into A; the gradient copies it to C (the splat's float atomics are its costliest launch).  K S(wn Q)
    // from A with B as scratch; K^T S(wn Q) from C with whichever of A / B the first result left free
    DSRG_LAUNCH(e, T_CRF_ENERGY, s,
                k_mf_zero<MP><<<bgrid, kThreads, 0, s>>>((float4 *)e->spA, e->sp.rowbase, (float4 *)e->biA,
                                                         e->bi.rowbase, B));
    DSRG_LAUNCH(e, T_CRF_ENERGY, s, k_kg_splatq<MP><<<gp, kThreads, 0, s>>>(ka, q, (float4 *)e->spA, (float4 *)e->biA));
    if (bwd)
        DSRG_LAUNCH(e, T_CRF_ENERGY, s,
                    k_crf_energy_copy<MP><<<bgrid, kThreads, 0, s>>>((const float4 *)e->spA, (float4 *)e->spC,
                                                                     e->sp.rowbase, (const float4 *)e->biA,
                                                                     (float4 *)e->biC, e->bi.rowbase, B));
    const float *vf_sp = blur_all<MP>(e, e->sp, e->spA, e->spB, nullptr, B, T_CRF_ENERGY, bgrid, s);
    const float *vf_bi = blur_all<MP>(e, e->bi, e->biA, e->biB, nullptr, B, T_CRF_ENERGY, bgrid, s);
    const float *vt_sp = nullptr, *vt_bi = nullptr;
    if (bwd) {
        vt_sp = blur_all<MP>(e, e->sp, e->spC, vf_sp == e->spA ? e->spB : e->spA, nullptr, B, T_CRF_ENERGY, bgrid, s,
                             true);
        vt_bi = blur_all<MP>(e, e->bi, e->biC, vf_bi == e->biA ? e->biB : e->biA, nullptr, B, T_CRF_ENERGY, bgrid, s,
                             true);
    }
    const float4 *a0 = (const float4 *)vf_sp, *a1 = (const float4 *)vf_bi;
    const float4 *a2 = (const float4 *)vt_sp, *a3 = (const float4 *)vt_bi;
    if (bwd && compat)
        DSRG_LAUNCH(e, T_CRF_ENERGY, s, (k_crf_energy<MP, true, true><<<gp, kThreads, 0, s>>>(ea, a0, a1, a2, a3)));
    else if (bwd)
        DSRG_LAUNCH(e, T_CRF_ENERGY, s, (k_crf_energy<MP, false, true><<<gp, kThreads, 0, s>>>(ea, a0, a1, a2, a3)));
    else if (compat)
        DSRG_LAUNCH(e, T_CRF_ENERGY, s, (k_crf_energy<MP, true, false><<<gp, kThreads, 0, s>>>(ea, a0, a1, a2, a3)));
    else
        DSRG_LAUNCH(e, T_CRF_ENERGY, s, (k_crf_energy<MP, false, false><<<gp, kThreads, 0, s>>>(ea, a0, a1, a2, a3)));
    if (!bwd) DSRG_LAUNCH(e, T_CRF_ENERGY, s, k_crf_energy_reduce<<<B, 32, 0, s>>>(e->en_part, ka.nblk, terms));
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int meanfield_energy(Engine *e, int B, const float *q, const float *unary, const float *potts, const float *compat,
                     const dsrg_crf_params &p, float *terms, const float *grad_terms, float *grad_q, float *grad_unary,
                     cudaStream_t s) {
    switch (e->MP) {
#define DSRG_CASE(MPV) \
    case MPV: return energy_impl<MPV>(e, B, q, unary, potts, compat, p, terms, grad_terms, grad_q, grad_unary, s);
        DSRG_CASE(4) DSRG_CASE(8) DSRG_CASE(12) DSRG_CASE(16) DSRG_CASE(20) DSRG_CASE(24) DSRG_CASE(28) DSRG_CASE(32)
#undef DSRG_CASE
    }
    set_error("unsupported label count %d", e->M);
    return DSRG_E_INVALID;
}

}  // namespace dsrg
