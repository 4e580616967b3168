// Shared declarations of the H100-native DSRG hot path (internal; the public surface is
// include/dsrg_b200.h).  sm_90a only.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <map>
#include <string>
#include <vector>

#include "../../include/dsrg_b200.h"

namespace dsrg {

constexpr int kThreads = 256;
constexpr uint64_t kEmptyKey = 0xFFFFFFFFFFFFFFFFull;
constexpr float kMinProb = 0.0001f;  // pylayers/pylayers/pylayers.py:20

void set_error(const char *fmt, ...);

#define DSRG_CUDA_TRY(expr)                                                              \
    do {                                                                                 \
        cudaError_t _e = (expr);                                                         \
        if (_e != cudaSuccess) {                                                         \
            dsrg::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),      \
                            __FILE__, __LINE__);                                         \
            return DSRG_E_CUDA;                                                          \
        }                                                                                \
    } while (0)

inline int cdiv(long long a, int b) { return (int)((a + b - 1) / b); }

// One permutohedral lattice family (spatial d=2 shared by the batch, or bilateral d=5 per image).
// Value rows: image b owns rows [rowbase[b], rowbase[b+1]); the first one is an all-zero row
// that stands for "missing neighbour" (the reference shifts ids by +1 for the same purpose,
// CRF/src/permutohedral.cpp:478-479, :534).
struct Lattice {
    int d = 0;
    int shared = 0;         // 1: one structure (image 0) reused by every image of the batch
    int nimg = 0;           // structures held (1 if shared, else max_batch)
    int N = 0;              // pixels
    int P = 0;              // phantom lanes (permutohedral.cpp:196: tail of the last 4-block)
    int cap = 0;            // hash slots per structure
    int capv = 0;           // max vertices per structure = (N+P)*(d+1)
    long long rows_cap = 0; // rows in the value buffers (all images)
    long long slots_alloc = 0, verts_alloc = 0;  // hkeys / hval and vkey entries allocated (capacity shape, all structures)
    int32_t *off = nullptr;     // [nimg][d+1][N] local row (1-based; 0 = zero row)
    float *bary = nullptr;      // [nimg][d+1][N]
    float *norm = nullptr;      // [nimg][N]
    uint64_t *hkeys = nullptr;  // [nimg][cap]
    int32_t *hval = nullptr;    // [nimg][cap] local vertex id of the slot
    int32_t *vslot = nullptr;   // [nimg][capv] slot of local vertex id
    int32_t *vcount = nullptr;  // [nimg]
    // build scratch of the renumbering (lattice.cu): the slot and the key (first incidence) of each vertex in
    // arrival order (vkey is kNoKey between builds), the key-space bitmap with its per-word prefix, and the
    // per-chunk prefix
    int32_t *aslot = nullptr;   // [nimg][capv]
    int32_t *vkey = nullptr;    // [nimg][capv]
    uint2 *rn_words = nullptr;  // [nimg][renum_words()]
    int32_t *rn_chunk = nullptr;  // [nimg][renum_words() / chunk]
    int32_t *rowbase = nullptr; // [max_batch+1]
    int2 *nbr = nullptr;        // [d+1][rows] (n1,n2): global rows (per-image) or local rows (shared)
    long long nbr_stride = 0;   // rows per axis in nbr
    // tile-local view (32x8-pixel tiles): the distinct vertices a tile touches, so that splat and
    // slice run out of shared memory (see tiles.cu)
    int maxloc = 0;                // local-vertex capacity per tile (kMaxLocSp / kMaxLocHy)
    int32_t *tl_nloc = nullptr;    // [nimg][ntiles] local vertices of the tile; | kTileHybrid: hybrid tile; -1: overflow tile without a list
    uint8_t *tl_hy = nullptr;      // [nimg][ntiles] 1: hybrid tile, k_mf_tile skips it (bilateral only)
    int2 *tl_hdr = nullptr;        // [nimg][ntiles][maxloc] per local vertex: (first entry | count<<16, local row id)
    uint16_t *tl_pack = nullptr;   // [nimg][ntiles][entcap] CSR entries grouped by local vertex:
                                   // r << 8 | pixel's thread index in the tile (see kEntZero)
    int entcap = 0;                // 256*(d+1) + maxloc, a multiple of 8 (16-byte blocks for the bulk copy)
    uint16_t *tl_loc = nullptr;    // [nimg][d+1][N] local vertex index of (pixel, r), kLocRemote if not in the tile's list
    float *wn = nullptr;           // [nimg][d+1][N] barycentric weight * norm
    // the same two per tile, in the order the forward tile kernels keep them in shared memory (one bulk copy each):
    // [nimg][ntiles][d+1][kTileThreads], slot t = the tile's pixel t; outside the image weight 0 and kLocRemote
    float *tl_w = nullptr;
    uint16_t *tl_li = nullptr;
    float scale[5] = {0, 0, 0, 0, 0};  // elevation scale factors (permutohedral.cpp:179-182)
    float sigma[5] = {0, 0, 0, 0, 0};  // feature sigmas: x, y[, c0, c1, c2]
};

struct Engine;

// kernel classes for the optional per-kernel CUDA-event timing (bench.py's roofline leg)
enum KTag {
    T_LAT_INSERT = 0, T_LAT_MISC, T_LAT_NORM, T_MF_INIT, T_MF_ZERO, T_MF_BLUR_SP,
    T_MF_BLUR_BI, T_MF_TILE, T_MF_EXPORT, T_SRG_LABEL, T_SRG_MERGE, T_SRG_FLAG, T_SRG_EMIT,
    T_LOSS, T_WIRE, T_PREP, T_POST, T_ANNOT, T_MF_TILE_HY, T_KGRAD, T_FGRAD, T_WIDE_GRAD, T_CRF_ENERGY, T_COUNT
};

// ---- lattice.cu ----
// feat ([B][5][N], bilateral lattice only): caller-given features in place of the image's; a key outside the packed
// range sets bad[b] (the engine's error flag is left alone)
int lattice_build(Engine *e, Lattice &L, int B, const uint8_t *image_dev, cudaStream_t s, const float *feat = nullptr,
                  int *bad = nullptr);
constexpr int kNoKey = 0x7F7F7F7F;  // renumbering key of no incidence yet (a byte pattern, for cudaMemset)
constexpr int kRenumChunk = 4 * kThreads;  // bitmap words per renumbering chunk: 4 per thread of k_renum_scan
long long renum_words(int ntiles, int dp1);  // bitmap words per image, a whole number of chunks
// what a build must leave for the next one, over every structure's whole allocation: counts[0] hash slots that are
// not kEmptyKey, [1] hval entries that are not -1, [2] vkey entries that are not kNoKey (synchronises the device)
int lattice_idle(Engine *e, const Lattice &L, long long *counts);
// ---- tiles.cu ----
constexpr int kTileW = 32, kTileH = 8;   // one thread per pixel, one warp per tile row
constexpr int kTileThreads = kTileW * kTileH;
#ifndef DSRG_MAXLOC_BI
#define DSRG_MAXLOC_BI 192
#endif
#ifndef DSRG_TILE_CTAS
#define DSRG_TILE_CTAS 4
#endif
#ifndef DSRG_SPLAT_UNROLL
#define DSRG_SPLAT_UNROLL 8
#endif
// Rows staged in the tile kernel's shared memory (lattice value rows, then the tile's Q rows) are padded by
// DSRG_ROW_PAD float4: with M = 21 the stride becomes 112 instead of 96 bytes, so the 8 rows a quarter-warp
// touches in one 128-bit request fall into 8 different bank groups unless they are equal mod 8 (mod 4 before).
#ifndef DSRG_ROW_PAD
#define DSRG_ROW_PAD 1
#endif
#ifndef DSRG_MAXLOC_SP
#define DSRG_MAXLOC_SP 128
#endif
// hybrid tiles (more distinct bilateral vertices than DSRG_MAXLOC_BI) are run by their own kernel, k_mf_tile_hy,
// DSRG_HY_CTAS CTAs per SM with room for DSRG_MAXLOC_HY local vertices; the other incidences go direct
#ifndef DSRG_MAXLOC_HY
#define DSRG_MAXLOC_HY 256
#endif
#ifndef DSRG_HY_CTAS
#define DSRG_HY_CTAS 3
#endif
constexpr int kMaxLocSp = DSRG_MAXLOC_SP, kMaxLocBi = DSRG_MAXLOC_BI, kMaxLocHy = DSRG_MAXLOC_HY;
static_assert(kMaxLocHy >= kMaxLocBi, "a hybrid tile holds at least what a plain one does");
constexpr int kSplatUnroll = DSRG_SPLAT_UNROLL;
// tl_loc value of a (pixel, vertex) incidence that is NOT in the tile-local list, and the flag in tl_nloc of a tile
// that has such incidences (a hybrid tile, tiles.cu)
constexpr int kLocRemote = 0xFFFF, kTileHybrid = 1 << 16;
// A CSR entry (tl_pack) is 16 bits, r << 8 | t: t is the pixel's thread index in the tile (its Q row), r its
// incidence index in one index space for both lattices (spatial 0..2, bilateral 3..8).  The mean-field kernels
// keep the weights of the current tile in a shared table wtab[r][kTileThreads], so the entry indexes it directly;
// the padding entry that evens a segment out points at the table's zero slot.
static_assert(kTileThreads == 256, "the entry's low byte is the thread index");
constexpr int kEntRows = 9;
constexpr int kEntZero = kEntRows << 8;  // wtab[kEntZero] = 0; its Q row (t = 0) is a valid one
__host__ __device__ constexpr int ent_r0(int dp1) { return dp1 == 3 ? 0 : 3; }  // first r of a lattice
// an overflow tile becomes a hybrid one when its local list would cover at least this share (percent) of its
// incidences; below that (uniform-noise images, the sigma/12 training lattices) the plain direct path is faster
// ... and only when the batch has at least DSRG_HY_MIN_TILES hybrid tiles per SM (tiles.cu: k_tile_demote)
#ifndef DSRG_HY_MIN_TILES
#define DSRG_HY_MIN_TILES 8
#endif
#ifndef DSRG_HY_MIN_COVER
#define DSRG_HY_MIN_COVER 40
#endif
int tiles_build(Engine *e, Lattice &L, int nb, cudaStream_t s);
// hybrid tiles pay off only when the batch has enough tiles to keep the GPU busy: small passes (the 41x41 training
// shape: 240 tiles; one VOC-sized image: 800) are launch-bound -- the hybrid kernel's eleven extra launches would
// outweigh what it saves -- and every overflow tile stays on k_mf_tile's direct path
inline bool hybrid_tiles_on(const Engine *e, int B);
// ---- meanfield.cu ----
// The inference: Q_T to e->Q0.  `compat` ({mu_bi, mu_sp} [2][M][M], device) replaces the Potts weights of p.
int meanfield_run(Engine *e, int B, const float *unary, int unary_layout, bool clamp_inplace,
                  float *unary_rw, const dsrg_crf_params &p, cudaStream_t s, const float *compat = nullptr);
// One call of the differentiable CRF: the training forward (unary -> q_out) or its backward (q_hist, grad_q -> the
// grad_* outputs).  The bilateral lattice is the image's or the caller-given features'; the pairwise weights are
// potts {w1, w2} or compat {mu_bi, mu_sp} [2][M][M] (neither: the params' w1 / w2).  A NULL output is not written.
struct CrfTrainIo {
    const float *unary = nullptr;     // [B][M][N] NCHW
    const float *q_hist = nullptr;    // [T+1][B][M][N]: the forward's Q_0..Q_T
    const float *grad_q = nullptr;    // [B][M][N] dL/dQ_T
    const uint8_t *image = nullptr;   // [B][N][3]
    const float *features = nullptr;  // [B][5][N]
    const float *potts = nullptr;
    const float *compat = nullptr;
    float *q_out = nullptr;           // the forward's Q_0..Q_T
    float *grad_unary = nullptr;      // [B][M][N]
    float *grad_potts = nullptr;      // [B][2] {dL/dw1, dL/dw2}
    float *grad_compat = nullptr;     // [B][2][M][M]
    float *grad_theta = nullptr;      // [B][7] dL/dtheta in dsrg_crf_params' order (image lattice only)
    float *grad_features = nullptr;   // [B][5][N] dL/df
    float *grad_theta_sp = nullptr;   // [B][2] dL/dtheta_gamma (features only)
};
// the training forward and its backward; at most DSRG_MAX_LABELS labels.  The backward needs e->compat_part with
// compat (ensure_compat_part), and the kg_* buffers (ensure_kgrad) with grad_theta or features.
int meanfield_run_train(Engine *e, int B, const CrfTrainIo &io, const dsrg_crf_params &p, cudaStream_t s);
int meanfield_backward(Engine *e, int B, const CrfTrainIo &io, const dsrg_crf_params &p, cudaStream_t s);
// NaN into every image b of p ([reps][B][per_image] floats) with bad[b] set; timed under tag
void nan_images(Engine *e, const int *bad, float *p, int B, long long per_image, int reps, cudaStream_t s, int tag);
// The energy of given marginals q [B][M][N] (DenseCRF::klDivergence) on the lattices the pass just built, at most
// DSRG_MAX_LABELS labels: terms [B][4] {entropy, unary, spatial, bilateral} or, with grad_terms [B][4], its gradient
// grad_q [B][M][N] and, if given, grad_unary.  unary may be nullptr; potts {w1, w2} or compat {mu_bi, mu_sp} [2][M][M]
// (neither: p's w1 / w2).  Needs e->en_part (ensure_energy); uses the mean-field value buffers.
int meanfield_energy(Engine *e, int B, const float *q, const float *unary, const float *potts, const float *compat,
                     const dsrg_crf_params &p, float *terms, const float *grad_terms, float *grad_q, float *grad_unary,
                     cudaStream_t s);
// the backward's per-image parameter sums, in a fixed order: part [B][nparts] {spatial, bilateral} -> out [B][2]
// {dL/dw1, dL/dw2}; part [B][nparts][mm2] -> out [B][mm2] = -sum over the parts
void potts_reduce(Engine *e, const float2 *part, float *out, int nparts, int B, int tag, cudaStream_t s);
void compat_reduce(Engine *e, const float *part, float *out, int nparts, int mm2, int B, int tag, cudaStream_t s);
// ---- meanfield_wide.cu: label counts above DSRG_MAX_LABELS ----
int meanfield_run_wide(Engine *e, int B, const float *unary, int unary_layout, bool clamp_inplace,
                       float *unary_rw, const dsrg_crf_params &p, cudaStream_t s, const float *compat);
int wide_weights(Engine *e, Lattice &L, int nb, cudaStream_t s);
// the training forward and its backward above DSRG_MAX_LABELS labels, as meanfield_run_train / meanfield_backward
// (potts or compat, not both); the backward needs e->wide_ppart, and with compat e->wide_g and e->wide_cpart
// (ensure_wide).  The matrices' outer products are summed per image over kWideChunks fixed pixel chunks.  grad_theta
// or features need e->kg_csum, e->kg_part and the 4-wide e->kg_sp / e->kg_bi (ensure_kgrad_wide)
constexpr int kWideChunks = 16;
int meanfield_run_train_wide(Engine *e, int B, const CrfTrainIo &io, const dsrg_crf_params &p, cudaStream_t s);
int meanfield_backward_wide(Engine *e, int B, const CrfTrainIo &io, const dsrg_crf_params &p, cudaStream_t s);
// meanfield_energy above DSRG_MAX_LABELS labels, with the same arguments and buffers (e->en_part); it also overwrites
// e->U and e->Q0 (the matrices' planes)
int meanfield_energy_wide(Engine *e, int B, const float *q, const float *unary, const float *potts, const float *compat,
                          const dsrg_crf_params &p, float *terms, const float *grad_terms, float *grad_q,
                          float *grad_unary, cudaStream_t s);
// (meanfield.cu) per image: the energy's block sums part [B][nblk][4] in block order -> terms [B][4]; <<<B, 32>>>
__global__ void k_crf_energy_reduce(const double *part, int nblk, float *terms);
int meanfield_export(Engine *e, int B, float *out, int layout, cudaStream_t s);
int meanfield_export_map(Engine *e, int B, int32_t *labels, cudaStream_t s);
int meanfield_export_renorm(Engine *e, int B, float *result_out, float *log_out, cudaStream_t s);
// ---- srg.cu ----
int srg_run(Engine *e, int B, const float *labels, const float *probs, const float *cues,
            double th1, double th2, int renorm, float *seeds_out, int32_t *label_map_out,
            cudaStream_t s, const uint32_t *cue_bits = nullptr, uint32_t *seed_bits = nullptr);
// ---- api.cu: the full pass with optional 1-bit cue / seed planes (wire.cu), and the CRF of a pass's body ----
int dsrg_forward_core(Engine *e, int B, const float *labels, float *probs, const float *cues, const uint32_t *cue_bits,
                      const uint8_t *image, const dsrg_crf_params *params, double th1, double th2, float *seeds_out,
                      uint32_t *seed_bits, float *crf_out, cudaStream_t s);
// The learned CRF at inference (dsrg_crf_batch_learned_dev, dsrg_predict_mask_batch_learned_dev): caller-given
// bilateral features ([B][5][N], in place of the image; they need e->feat_bad, ensure_feat) and / or the matrices
// ({mu_bi, mu_sp} [2][M][M]).  An image whose feature lattice leaves the packed key range gets NaN marginals in e->Q0.
struct LearnedCrf {
    const float *features, *compat;
};
int crf_core(Engine *e, int B, const float *unary, int layout, bool clamp, float *unary_rw, const uint8_t *image,
             const dsrg_crf_params *p, cudaStream_t s, const LearnedCrf *lc = nullptr);
int ensure_feat(Engine *e);
// ---- sec_loss.cu ----
constexpr int kSecPlainChunks = 16;  // CTAs per image of SeedLossLayer's sums (fixed, so is their order)

struct Engine {
    int device = 0;
    int numa_node = -1;  // node of the GPU when host-side placement is on (numa.cu), else -1
    int maxB = 0, H = 0, W = 0, M = 0, MP = 0, N = 0;
    int Hcap = 0, Wcap = 0, Ncap = 0;  // shape the buffers were sized for (H <= Hcap, W <= Wcap)
    int sm_count = 132;
    size_t bytes = 0;
    long long launches = 0;

    Lattice sp, bi;
    bool sp_valid = false;

    // mean-field state, planar [B][M][N]
    float *U = nullptr, *Q0 = nullptr;
    int last_crf_B = 0;    // images whose raw marginals of the last mean-field pass are still in Q0 (0: none)
    // lattice value buffers [rows][MP]
    float *spA = nullptr, *spB = nullptr, *spC = nullptr, *biA = nullptr, *biB = nullptr, *biC = nullptr;
    int tiles_x = 0, tiles_y = 0, ntiles = 0;  // tiles of tile_w x 8 pixels
    int tile_w = 32;  // <= 32: the image width is split evenly so that no sliver tiles remain
    int2 *hy_list = nullptr;   // [maxB * ntiles] (tile, image) of the hybrid tiles of the current lattices
    float2 *potts_part = nullptr;  // [maxB * ntiles] the CRF backward's per-tile Potts partials (spatial, bilateral)
    // [maxB * ntiles][2][M][M] the compatibility backward's per-tile partials (bilateral, spatial); allocated by its
    // first call (ensure_compat_part)
    float *compat_part = nullptr;
    // the kernel-bandwidth backward's buffers, allocated by its first call (ensure_kgrad): g_t [maxB][M][N], c per
    // pixel [2][maxB][N], per-block sums [maxB][blocks][8], and two value buffers per lattice [rows][MP].  Above
    // DSRG_MAX_LABELS (ensure_kgrad_wide) there is no kg_g, and the value buffers are [rows][4]: the label-chunked
    // backward uses them only for the normalisation term
    float *kg_g = nullptr, *kg_csum = nullptr, *kg_part = nullptr;
    float *kg_sp[2] = {nullptr, nullptr}, *kg_bi[2] = {nullptr, nullptr};
    // the feature passes' per-image key-range flags [maxB] (allocated by the first one) and that pass's batch
    int *feat_bad = nullptr;
    int feat_B = 0;
    // the label-chunked backward's buffers, allocated by its first call (ensure_wide): the Potts partials
    // [maxB][MP/4][blocks] float2, and for matrices G [maxB][M][N] and the outer-product partials
    // [maxB][kWideChunks][2][M][M]
    float2 *wide_ppart = nullptr;
    float *wide_g = nullptr, *wide_cpart = nullptr;
    int *hy_count = nullptr;   // their number (device-resident)
    // the energy's per-block sums [maxB][blocks][4], allocated by its first call (ensure_energy)
    double *en_part = nullptr;
    // 1-channel buffers for the normalisation pass
    float *nvA = nullptr, *nvB = nullptr;
    // SRG state
    uint8_t *lmap = nullptr;   // [B][N] label map value (0 = none, c+1)
    uint8_t *lflag = nullptr;  // [B][N] bit0 own-seed, bit1 excluded
    int32_t *parent = nullptr; // [B][N] union-find forest
    uint8_t *hc = nullptr;     // [B][N] high-confidence flag per root
    // loss scratch
    double *loss_acc = nullptr;  // [B][4]
    // SEC losses (sec_loss.cu): per-plane GWRP records, per-image sums, SeedLoss partials, the q^i tables
    double2 *sec_rec = nullptr;   // [B][M] (G, max)
    double *sec_img = nullptr;    // [B][3]
    double2 *sec_part = nullptr;  // [B][kSecPlainChunks]
    double *sec_w = nullptr;      // [2][sec_wcap]: q_fg table, then q_bg table
    int sec_wcap = 0;             // min(Ncap, DSRG_GWRP_MAX_PLANE)
    double sec_q[2] = {0, 0}, sec_z[2] = {0, 0};
    int sec_n[2] = {0, 0};        // (q, n) the device tables hold; 0 = none yet
    std::vector<double> sec_w_host[2];
    // staging for the *_host entry points
    float *st_unary = nullptr, *st_out = nullptr, *st_cues = nullptr, *st_labels = nullptr;
    uint8_t *st_image = nullptr;
    int32_t *st_sel = nullptr;  // [M] label selection of dsrg_predict_mask_*, written by its pass (post.cu)
    // staging whose size depends on the call, grown on demand (grow_staging); capacities in bytes
    float *st_raw = nullptr;   // raw (un-zoomed) images and score maps of the *_host entry points
    size_t st_raw_cap = 0;
    int32_t *st_idx = nullptr;  // index lists of the annotation entry points
    size_t st_idx_cap = 0;
    uint8_t *st_prep = nullptr;  // image and network inputs of dsrg_prepare_net_input_host
    size_t st_prep_cap = 0;
    int32_t *st_lmap = nullptr;
    cudaStream_t own_stream = nullptr, in_stream = nullptr, out_stream = nullptr;
    // order of the passes of this engine across streams (StreamScope)
    cudaEvent_t order_event = nullptr;
    cudaStream_t last_stream = nullptr;
    bool last_stream_valid = false;
    std::vector<cudaEvent_t> pipe_events;
    int host_chunk = 0;   // > 0 caps the images per pipeline stage of the *_host entry points
    // 0/1 planes travel over PCIe as bit masks (wire.cu): device + pinned host staging, [maxB][words/image]
    uint32_t *d_cbits = nullptr, *d_sbits = nullptr, *d_mbits = nullptr;
    uint32_t *h_cbits = nullptr, *h_sbits = nullptr, *h_mbits = nullptr;
    int wire_compress = 1;
    int *dev_err = nullptr;  // device-side error flag
    // CUDA graphs of whole device passes, keyed by everything a pass's launch arguments depend on (graph.cu)
    struct GraphRec { cudaGraphExec_t exec = nullptr; long long launches = 0; unsigned long long last_use = 0; bool bad = false; };
    std::map<std::string, GraphRec> graphs;
    unsigned long long graph_clock = 0;
    int use_graphs = 1;
    long long graph_replays = 0;
    // per-kernel event timing (off by default)
    bool prof = false;
    struct ProfRec { int tag; cudaEvent_t a, b; };
    std::vector<ProfRec> prof_recs;
    std::vector<cudaEvent_t> prof_pool;
};

// An engine is one set of buffers: two passes must not overlap.  Passes issued on ONE stream are ordered by it;
// when a caller moves to another stream (torch side streams are non-blocking: not even the legacy default stream
// orders them) the new pass first waits for the event the previous pass left behind.  Costs one cudaEventRecord
// per entry point.  Inside the caller's own stream capture nothing is recorded or awaited.
struct StreamScope {
    Engine *e;
    cudaStream_t s;
    bool live = false;
    StreamScope(Engine *e_, cudaStream_t s_) : e(e_), s(s_) {
        if (!e || !e->order_event) return;
        cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(s, &st) != cudaSuccess) {
            cudaGetLastError();
            return;
        }
        if (st != cudaStreamCaptureStatusNone) return;
        live = true;
        if (e->last_stream_valid && e->last_stream != s && cudaStreamWaitEvent(s, e->order_event, 0) != cudaSuccess)
            cudaGetLastError();
    }
    ~StreamScope() {
        if (!live) return;
        if (cudaEventRecord(e->order_event, s) == cudaSuccess) {
            e->last_stream = s;
            e->last_stream_valid = true;
        } else {
            cudaGetLastError();
        }
    }
};

inline bool hybrid_tiles_on(const Engine *e, int B) {
    return e->MP <= DSRG_MAX_LABELS && (long long)e->ntiles * B >= 16LL * e->sm_count;
}

// RAII bracket around one kernel launch: counts it and, when profiling is on, times it with a pair
// of CUDA events on the launching stream.
struct LaunchScope {
    Engine *e;
    cudaStream_t s;
    cudaEvent_t b = nullptr;
    LaunchScope(Engine *e_, int tag, cudaStream_t s_) : e(e_), s(s_) {
        e->launches++;
        if (e->prof) {
            cudaEvent_t a = take();
            b = take();
            cudaEventRecord(a, s);
            e->prof_recs.push_back({tag, a, b});
        }
    }
    ~LaunchScope() {
        if (b) cudaEventRecord(b, s);
    }
    cudaEvent_t take() {
        if (!e->prof_pool.empty()) {
            cudaEvent_t ev = e->prof_pool.back();
            e->prof_pool.pop_back();
            return ev;
        }
        cudaEvent_t ev;
        cudaEventCreate(&ev);
        return ev;
    }
};
#define DSRG_LAUNCH(e, tag, s, ...)          \
    do {                                     \
        dsrg::LaunchScope _ls((e), (tag), (s)); \
        __VA_ARGS__;                         \
    } while (0)


// float64 sum of n values in the order NumPy adds a contiguous reduction axis (pairwise_sum in
// numpy/core/src/umath/loops_utils.h.src: eight accumulators, their fixed combination tree, then the tail;
// blocks of at most 128).  The reference renormalises with np.sum(result, axis=1) on a TRANSPOSED view of an
// (N,H,W,C) float64 array (pylayers.py:328-330, :85-86), i.e. the class axis is the contiguous one and this is
// the order its sum is formed in; for 21 classes it differs from a sequential sum in the last bit on ~17 % of
// the pixels, which matters to the strict float64 threshold compares that follow (pylayers.py:251-257).
// `get(i)` returns element i; NT > 0 makes n a compile-time constant.
template <int NT, typename F>
__device__ __forceinline__ double numpy_sum_block(F get, int lo, int n_rt) {
    const int n = NT ? NT : n_rt;
    if (n < 8) {
        double res = 0.0;
#pragma unroll
        for (int i = 0; i < n; i++) res += get(lo + i);
        return res;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; j++) r[j] = get(lo + j);
    int i = 8;
#pragma unroll
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; j++) r[j] += get(lo + i + j);
    }
    double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
#pragma unroll
    for (; i < n; i++) res += get(lo + i);
    return res;
}
template <int NT, typename F>
__device__ __forceinline__ double numpy_sum(F get, int n_rt) {
    const int n = NT ? NT : n_rt;
    if (n <= 128) return numpy_sum_block<NT>(get, 0, n);
    // n <= 255 here (DSRG_MAX_LABELS_WIDE, SRG's 255).  NumPy splits at n/2 rounded down to a multiple of 8 and
    // recurses into both halves: the first (<= 127) is one block, the second (<= 135) is split once more when it
    // exceeds 128, which happens from n = 249 on
    int n2 = n / 2;
    n2 -= n2 % 8;
    const double lo = numpy_sum_block<0>(get, 0, n2);
    const int m = n - n2;
    if (m <= 128) return lo + numpy_sum_block<0>(get, n2, m);
    int m2 = m / 2;
    m2 -= m2 % 8;
    return lo + (numpy_sum_block<0>(get, n2, m2) + numpy_sum_block<0>(get, n2 + m2, m - m2));
}

// Entry points run on the engine's device and hand the calling thread back on the device it came with: a Caffe
// solver thread (or any host framework) keeps its own current device across a drop-in call.
struct DeviceScope {
    int prev = -1;
    bool switched = false;
    explicit DeviceScope(const Engine *e) : DeviceScope(e ? e->device : -1) {}
    explicit DeviceScope(int device) {  // device < 0: nothing to select
        if (device < 0) return;
        if (cudaGetDevice(&prev) != cudaSuccess) {
            cudaGetLastError();
            prev = -1;
        }
        if (prev != device) switched = cudaSetDevice(device) == cudaSuccess && prev >= 0;
    }
    ~DeviceScope() {
        if (switched) cudaSetDevice(prev);
    }
    DeviceScope(const DeviceScope &) = delete;
    DeviceScope &operator=(const DeviceScope &) = delete;
};

// ---- numa.cu: host-side placement for one-process-per-GPU jobs ----
bool numa_wanted();
int numa_node_of_device(int device);
bool numa_bind_thread(int node);
bool numa_prefer_memory(int node);
cudaError_t numa_host_alloc(void **p, size_t bytes, int device);

// ---- graph.cu: replay a device pass as one CUDA graph ----
// A pass (lattice build + mean-field loop + SRG ...) is 40-130 dependent launches whose arguments depend only on
// the call's arguments; `key` holds all of them.  First sighting of a key: run eagerly.  Second: capture the same
// launches from the stream into a graph, instantiate, launch.  Afterwards: one cudaGraphLaunch.  Falls back to
// plain launches on the legacy default stream, inside somebody else's capture, while per-kernel profiling is on,
// or if capture fails.  `body` issues the launches on `s` and returns a DSRG_* code.
enum class PassKind : int { crf, crf_map, forward, crflayer, densecrf, post, crf_train, crf_backward, crf_train_compat,
                            crf_backward_compat, crf_backward_theta, crf_backward_compat_theta, crf_train_feat,
                            crf_backward_feat, crf_train_wide, crf_backward_wide, crf_backward_wide_theta,
                            crf_train_wide_feat, crf_backward_wide_feat, crf_learned, post_learned, crf_energy,
                            crf_energy_backward, crf_energy_wide, crf_energy_backward_wide };
struct GraphKey {
    std::string bytes;
    GraphKey() = default;
    // the key of a pass: its kind, its batch and the image size, then the call's own arguments
    GraphKey(PassKind kind, int B, const Engine *e, const GraphKey &args) {
        add(kind).add(B).add(e->H).add(e->W);
        bytes += args.bytes;
    }
    template <typename T>
    GraphKey &add(const T &v) {
        bytes.append(reinterpret_cast<const char *>(&v), sizeof(T));
        return *this;
    }
};
constexpr int kGraphRetry = 1;  // graph_end: the capture could not be turned into a graph, issue the launches again
int graph_begin(Engine *e, cudaStream_t s, const GraphKey &key, bool *captured);   // 1: replayed (skip body), 0: run body
int graph_end(Engine *e, cudaStream_t s, const GraphKey &key, bool captured, int body_rc, long long launches_before);
void graph_clear(Engine *e);
template <typename F>
inline int run_pass(Engine *e, cudaStream_t s, const GraphKey &key, bool allow_graph, F body) {
    if (!allow_graph) return body();
    bool cap = false;
    const long long l0 = e->launches;
    const int g = graph_begin(e, s, key, &cap);
    if (g != 0) return g < 0 ? g : DSRG_OK;
    int rc = body();
    if (!cap) return rc;
    rc = graph_end(e, s, key, cap, rc, l0);
    if (rc == kGraphRetry) {
        e->launches = l0;
        rc = body();
    }
    return rc;
}

// ---- api.cu: the host side of crf_pass ----
bool crf_pass_begin(Engine *e, const dsrg_crf_params &p);  // true: the pass rebuilds the shared spatial lattice
void crf_pass_end(Engine *e, const dsrg_crf_params &p, int B, int rc);

// Every mean-field pass runs through here; `args` are the call's own arguments.  The shared spatial lattice is rebuilt
// when the image size or its sigmas changed since it was built, and that rebuild is captured with the pass (`rebuild`
// is part of the key), so a graph is valid whatever the engine ran in between: the per-image callers alternate sizes
// and would otherwise never replay.  A replay skips the host code of `body`, so the notes it leaves (the spatial
// lattice's sigmas, the batch whose marginals Q0 holds) are written here, after the pass.
template <typename F>
inline int crf_pass(Engine *e, cudaStream_t s, PassKind kind, int B, const dsrg_crf_params *p, const GraphKey &args,
                    F body) {
    const bool rebuild = crf_pass_begin(e, *p);
    GraphKey key(kind, B, e, args);
    key.add(*p).add(rebuild);
    const int rc = run_pass(e, s, key, true, body);
    crf_pass_end(e, *p, B, rc);
    return rc;
}

int device_alloc(Engine *e, void **p, size_t bytes);
int check_batch(Engine *e, int B);
int ensure_staging(Engine *e);
int grow_staging(Engine *e, void **buf, size_t *cap_bytes, size_t bytes);  // frees the old buffer first
int check_device_flag(Engine *e, cudaStream_t s);
void wire_free(Engine *e);
template <typename T>
inline int dalloc(Engine *e, T **p, size_t count) {
    return device_alloc(e, (void **)p, count * sizeof(T));
}

// ---- the prologue of every engine entry point of the C ABI ----
// In this order: the engine's device for the whole call (DeviceScope, restored on every path), the NULL engine and
// the batch range (check_batch), the arguments, and only then the stream (StreamScope).  `args_ok` is false when a
// required pointer is NULL or a plain argument is out of range; a call rejected here allocates and queues nothing.
// Checks that need the engine's shape or labels stay in the body.
inline int check_entry(Engine *e, int B, bool args_ok) {
    if (int rc = check_batch(e, B)) return rc;
    if (args_ok) return DSRG_OK;
    set_error("bad argument (NULL pointer or value out of range)");
    return DSRG_E_INVALID;
}

// *_dev entry points: body(e) runs on the caller's stream `s`
template <typename F>
inline int dev_call(dsrg_engine *h, int B, cudaStream_t s, bool args_ok, F body) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    if (int rc = check_entry(e, B, args_ok)) return rc;
    StreamScope stream_scope(e, s);
    return body(e);
}

// *_host entry points: the same prologue, then `state` (a check of what the engine holds, if given), the staging
// buffers (ensure_staging), and body(e, s) on the engine's own stream, which copies in, runs what the *_dev twin runs
// and copies out.  Returns once those copies have landed: through check_device_flag for the passes that end in it
// (`flag`), else a stream synchronisation.
template <typename F>
inline int host_call(dsrg_engine *h, int B, bool args_ok, bool flag, F body,
                     int (*state)(const Engine *, int) = nullptr) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_entry(e, B, args_ok);
    if (!rc && state) rc = state(e, B);
    if (rc || (rc = ensure_staging(e))) return rc;
    cudaStream_t s = e->own_stream;
    StreamScope stream_scope(e, s);
    if ((rc = body(e, s))) return rc;
    if (flag) return check_device_flag(e, s);
    DSRG_CUDA_TRY(cudaStreamSynchronize(s));
    return DSRG_OK;
}

}  // namespace dsrg
