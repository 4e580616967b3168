// Seeded region growing for a whole batch (sm_90a).
//
// Replaces generate_seed_step (pylayers/pylayers/pylayers.py:237-275) and the pure-Python
// two-pass labeller it calls per class (pylayers/pylayers/CC_labeling_8.py:103-282).
//
// The reference runs one binary 8-connectivity labelling per present class; the class masks
// label_map == c+1 are disjoint, so ONE equal-label 8-connectivity union-find over the
// multi-valued label map gives the same components (SURVEY.md 3.3).  Everything is integer /
// comparison work, hence bit-exact against the reference:
//   K1 label map   : thresholds compared in float64 exactly like the reference's data
//   K2 merge       : per-pixel union with the W / NW / N / NE neighbour of equal label; horizontal
//                    runs are pre-linked with a warp ballot (neighbour voting) so that only run
//                    heads and vertical links touch the global forest
//   K3 flag        : components containing an own-class seed become "high confidence"
//   K4 emit        : seeds_out = cues OR (grown AND NOT excluded)
#include "common.cuh"

namespace dsrg {

__device__ __forceinline__ int uf_find(const int32_t *parent, int x) {
    const volatile int32_t *vp = parent;  // other threads hook roots concurrently
    int p = vp[x];
    while (p != x) {
        x = p;
        p = vp[x];
    }
    return x;
}

// lock-free union by minimum index (label equivalence), safe under concurrent unions
__device__ __forceinline__ void uf_union(int32_t *parent, int a, int b) {
    while (true) {
        a = uf_find(parent, a);
        b = uf_find(parent, b);
        if (a == b) return;
        if (a > b) {
            int t = a;
            a = b;
            b = t;
        }
        int old = atomicMin(parent + b, a);  // hook the larger root under the smaller
        if (old == b) return;
        b = old;  // somebody re-hooked b meanwhile: retry from there
    }
}

// K1 --------------------------------------------------------------------------------------------
// MT > 0: the label count is a compile-time constant, so all 2*MT loads of a pixel are issued before the
// first use (the kernel is a stream of 2*MT planes and was latency-bound);
// MT == 0: generic run-time loop.
#ifndef DSRG_SRG_LABEL_CTAS
#define DSRG_SRG_LABEL_CTAS 1
#endif
// cue planes come either as float32 (the reference's blobs) or as 1 bit per value (the host pipeline's wire format,
// wire.cu: bit c*N + i of image b's words): CB selects the reader
template <bool CB>
__device__ __forceinline__ float cue_at(const float *cues_f, const uint32_t *cues_b, size_t img_base_f, size_t img_base_w,
                                        int c, int N, int i) {
    if (!CB) return __ldg(cues_f + img_base_f + (size_t)c * N + i);
    const size_t g = (size_t)c * N + i;
    return (__ldg(cues_b + img_base_w + (g >> 5)) >> (g & 31)) & 1u ? 1.0f : 0.0f;
}

template <int MT, bool CB>
__global__ void __launch_bounds__(kThreads, DSRG_SRG_LABEL_CTAS)
k_srg_label(const float *__restrict__ labels, const float *__restrict__ probs, const float *__restrict__ cues,
            const uint32_t *__restrict__ cue_bits, int wpi,
            double th1, double th2, int renorm, uint8_t *lmap, uint8_t *lflag, int32_t *parent, uint8_t *hc,
            int32_t *label_map_out, int Mrt, int N, int W) {
    const int M = MT ? MT : Mrt;
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < N;
    int L = 0;
    if (in) {
        const float *lab = labels + (size_t)b * M;
        const float *pb = probs + (size_t)b * M * N + i;
        const size_t cbase_f = (size_t)b * M * N, cbase_w = (size_t)b * wpi;
        // One pass over the classes.  With renorm the reference divides every clamped value by the
        // float64 sum s (pylayers.py:328-330) before taking the arg-max over the PRESENT classes
        // (first index wins ties, pylayers.py:240-243).  IEEE division by a common positive s is
        // monotone and cannot merge two distinct float32-exact values (they differ by >= 2^-24
        // relative, the quotient rounds at 2^-53), so arg-max(v/s) == arg-max(v) with identical ties;
        // only the winner is divided.
        int cstar = -1;
        double best = 0.0, s = 0.0;
        float nseed = 0.0f;   // np.sum(seed_c[:, x, y]) (pylayers.py:268)
        float cue_at_L = 0.0f;
        float cuv[MT ? MT : 1], pv[MT ? MT : 1];
        if (MT) {
#pragma unroll
            for (int c = 0; c < (MT ? MT : 1); c++) {
                cuv[c] = cue_at<CB>(cues, cue_bits, cbase_f, cbase_w, c, N, i);
                pv[c] = __ldg(pb + (size_t)c * N);
            }
        }
        // float64 sum of the clamped values in NumPy's order (common.cuh:numpy_sum), formed on the fly when the label
        // count is a compile-time constant in [8, 128]: eight accumulators over the first MT - MT % 8 values, their
        // fixed combination tree, then the tail
        constexpr bool kInline = MT >= 8 && MT <= 128;
        constexpr int kBody = MT - MT % 8;
        double r8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int c = 0; c < M; c++) {
            const float cu = MT ? cuv[MT ? c : 0] : cue_at<CB>(cues, cue_bits, cbase_f, cbase_w, c, N, i);
            nseed += cu;
            if (cu > 0.0f) {  // seeds: the highest class index wins (pylayers.py:248-250)
                L = c + 1;
                cue_at_L = cu;
            }
            double v = (double)(MT ? pv[MT ? c : 0] : pb[(size_t)c * N]);
            if (renorm && v < 0.0001) v = 0.0001;
            if (kInline && renorm) {
                if (c < 8) r8[c & 7] = v;
                else if (c < kBody) r8[c & 7] += v;
                else {
                    if (c == kBody) s = ((r8[0] + r8[1]) + (r8[2] + r8[3])) + ((r8[4] + r8[5]) + (r8[6] + r8[7]));
                    s += v;
                }
            }
            if (lab[c] == 1.0f && (cstar < 0 || v > best)) {
                best = v;
                cstar = c;
            }
        }
        if (renorm) {
            if (kInline) {
                if (MT == kBody) s = ((r8[0] + r8[1]) + (r8[2] + r8[3])) + ((r8[4] + r8[5]) + (r8[6] + r8[7]));
            } else {
                auto clamped = [&](int c) {
                    const double v = (double)(MT ? pv[MT ? c : 0] : pb[(size_t)c * N]);
                    return v < 0.0001 ? 0.0001 : v;
                };
                s = numpy_sum<MT>(clamped, M);
            }
            best = best / s;
        }
        // thresholds (pylayers.py:251-257): strict > in float64; overwrite the seed label
        if (cstar >= 0 && best > th2 && (cstar != 0 || best > th1)) {
            L = cstar + 1;
            cue_at_L = cue_at<CB>(cues, cue_bits, cbase_f, cbase_w, cstar, N, i);
        }
        uint8_t fl = 0;
        if (L > 0) {
            const bool present = lab[L - 1] == 1.0f;
            const bool own = cue_at_L == 1.0f;               // seed_c[c,x,y] == 1 (pylayers.py:266)
            if (present && own) fl |= 1;
            if (!own && nseed == 1.0f) fl |= 2;              // excluded (pylayers.py:268-269)
        }
        lmap[(size_t)b * N + i] = (uint8_t)L;
        lflag[(size_t)b * N + i] = fl;
        hc[(size_t)b * N + i] = 0;
        if (label_map_out) label_map_out[(size_t)b * N + i] = L;
    }
    // horizontal runs via warp ballot: a pixel links to the head of its run inside the warp's
    // 32-pixel window, so W-links never go through atomics
    const unsigned lane = threadIdx.x & 31;
    const int x = in ? i % W : 0;
    const int left = __shfl_up_sync(0xffffffffu, L, 1);
    const bool joins_left = in && lane > 0 && x > 0 && L > 0 && left == L;
    const unsigned brk = ~__ballot_sync(0xffffffffu, joins_left);  // bit set = run head
    if (in) {
        const unsigned below = brk & (0xffffffffu >> (31 - lane));  // heads at lanes <= mine
        const int head_lane = 31 - __clz(below);
        parent[(size_t)b * N + i] = i - ((int)lane - head_lane);
    }
}

// K2 --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_srg_merge(const uint8_t *lmap, int32_t *parent, int N, int W) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const uint8_t *lm = lmap + (size_t)b * N;
    int32_t *par = parent + (size_t)b * N;
    const int L = lm[i];
    if (L == 0) return;
    const int x = i % W;
    // W link across a warp-window boundary (inside the window the ballot already linked it)
    if (x > 0 && (threadIdx.x & 31) == 0 && lm[i - 1] == L) uf_union(par, i, i - 1);
    if (i >= W) {
        const int n = i - W;
        if (lm[n] == L) {
            // N covers NW and NE through the row above.  The link is redundant when the pixel to the left and the
            // one above it carry the same label: (i-1, n-1) then joins the same two horizontal runs -- by induction
            // the leftmost pixel of such a stretch makes the link, the rest skip their root chases
            if (!(x > 0 && lm[i - 1] == L && lm[n - 1] == L)) uf_union(par, i, n);
        } else {
            if (x > 0 && lm[n - 1] == L) uf_union(par, i, n - 1);
            if (x < W - 1 && lm[n + 1] == L) uf_union(par, i, n + 1);
        }
    }
}

// K3 --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_srg_flag(const uint8_t *lflag, int32_t *parent, uint8_t *hc, int N) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    int32_t *par = parent + (size_t)b * N;
    const int root = uf_find(par, i);
    par[i] = root;  // path compression for K4 (roots never change any more)
    if (lflag[(size_t)b * N + i] & 1) hc[(size_t)b * N + root] = 1;
}

// K4 --------------------------------------------------------------------------------------------
// seeds = cues OR (grown AND NOT excluded).  CB: cues are bits; SB: seeds are written as bits (into zeroed words:
// a warp's 32 pixels of one class are 32 consecutive bits that straddle at most two words -> two atomicOr by lane 0)
template <int MT, bool CB, bool SB>
__global__ void __launch_bounds__(kThreads)
k_srg_emit(const float *__restrict__ cues, const uint32_t *__restrict__ cue_bits, int wpi, const uint8_t *lmap,
           const uint8_t *lflag, const int32_t *parent, const uint8_t *hc, float *__restrict__ seeds_out,
           uint32_t *__restrict__ seed_bits, int Mrt, int N) {
    const int M = MT ? MT : Mrt;
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = i < N;
    if (!SB && !in) return;  // the bit writer needs whole warps for its ballots
    const size_t p = (size_t)b * N + (in ? i : 0);
    int grow_c = -1;
    if (in) {
        const int L = lmap[p];
        if (L > 0 && !(lflag[p] & 2)) {
            const int root = parent[p];  // fully compressed by K3
            if (hc[(size_t)b * N + root]) grow_c = L - 1;
        }
    }
    const size_t cbase_f = (size_t)b * M * N, cbase_w = (size_t)b * wpi;
    float *ob = seeds_out + (size_t)b * M * N + i;
    const int i0 = i & ~31;  // first pixel of this warp (blocks start at multiples of 256)
    if (MT) {
        float v[MT ? MT : 1];
#pragma unroll
        for (int c = 0; c < (MT ? MT : 1); c++) v[c] = in ? cue_at<CB>(cues, cue_bits, cbase_f, cbase_w, c, N, i) : 0.0f;
#pragma unroll
        for (int c = 0; c < (MT ? MT : 1); c++) {
            const float o = (c == grow_c) ? 1.0f : v[c];
            if (!SB) {
                ob[(size_t)c * N] = o;
            } else {
                const unsigned m = __ballot_sync(0xffffffffu, in && o != 0.0f);
                if ((threadIdx.x & 31) == 0 && m) {
                    const size_t g0 = (size_t)c * N + i0;
                    const int sh = (int)(g0 & 31);
                    atomicOr(seed_bits + cbase_w + (g0 >> 5), m << sh);
                    if (sh && (m >> (32 - sh))) atomicOr(seed_bits + cbase_w + (g0 >> 5) + 1, m >> (32 - sh));
                }
            }
        }
    } else {
        for (int c = 0; c < M; c++) {
            const float o = (c == grow_c) ? 1.0f : (in ? cue_at<CB>(cues, cue_bits, cbase_f, cbase_w, c, N, i) : 0.0f);
            if (!SB) {
                ob[(size_t)c * N] = o;
            } else {
                const unsigned m = __ballot_sync(0xffffffffu, in && o != 0.0f);
                if ((threadIdx.x & 31) == 0 && m) {
                    const size_t g0 = (size_t)c * N + i0;
                    const int sh = (int)(g0 & 31);
                    atomicOr(seed_bits + cbase_w + (g0 >> 5), m << sh);
                    if (sh && (m >> (32 - sh))) atomicOr(seed_bits + cbase_w + (g0 >> 5) + 1, m >> (32 - sh));
                }
            }
        }
    }
}

// cue_bits / seed_bits (optional): the planes in the host pipeline's 1-bit wire format (wpi words per image) instead of
// float32 -- saves expanding the cues to floats and packing the seeds again on the device
int srg_run(Engine *e, int B, const float *labels, const float *probs, const float *cues,
            double th1, double th2, int renorm, float *seeds_out, int32_t *label_map_out,
            cudaStream_t s, const uint32_t *cue_bits, uint32_t *seed_bits) {
    const int N = e->N, M = e->M;
    if (seed_bits && !cue_bits) {  // seeds keep every cue value: they are a 0/1 mask only when the cues are
        set_error("SRG seed bits need cue bits");
        return DSRG_E_INVALID;
    }
    const int wpi = (int)(((size_t)M * N + 31) / 32);
    dim3 g(cdiv(N, kThreads), B);
#define DSRG_LABEL(MTV, CBV)                                                                                          \
    DSRG_LAUNCH(e, T_SRG_LABEL, s,                                                                                     \
                (k_srg_label<MTV, CBV><<<g, kThreads, 0, s>>>(labels, probs, cues, cue_bits, wpi, th1, th2, renorm, e->lmap, \
                                                              e->lflag, e->parent, e->hc, label_map_out, M, N, e->W)))
    if (M == 21) { if (cue_bits) DSRG_LABEL(21, true); else DSRG_LABEL(21, false); }
    else { if (cue_bits) DSRG_LABEL(0, true); else DSRG_LABEL(0, false); }
#undef DSRG_LABEL
    DSRG_LAUNCH(e, T_SRG_MERGE, s, k_srg_merge<<<g, kThreads, 0, s>>>(e->lmap, e->parent, N, e->W));
    DSRG_LAUNCH(e, T_SRG_FLAG, s, k_srg_flag<<<g, kThreads, 0, s>>>(e->lflag, e->parent, e->hc, N));
    if (seed_bits) DSRG_CUDA_TRY(cudaMemsetAsync(seed_bits, 0, (size_t)B * wpi * sizeof(uint32_t), s));
#define DSRG_EMIT(MTV, CBV, SBV)                                                                                       \
    DSRG_LAUNCH(e, T_SRG_EMIT, s,                                                                                      \
                (k_srg_emit<MTV, CBV, SBV><<<g, kThreads, 0, s>>>(cues, cue_bits, wpi, e->lmap, e->lflag, e->parent, e->hc, \
                                                                  seeds_out, seed_bits, M, N)))
#define DSRG_EMIT_MT(MTV)                                              \
    if (cue_bits && seed_bits) DSRG_EMIT(MTV, true, true);             \
    else if (cue_bits) DSRG_EMIT(MTV, true, false);                    \
    else DSRG_EMIT(MTV, false, false)
    if (M == 21) { DSRG_EMIT_MT(21); } else { DSRG_EMIT_MT(0); }
#undef DSRG_EMIT_MT
#undef DSRG_EMIT
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

}  // namespace dsrg
