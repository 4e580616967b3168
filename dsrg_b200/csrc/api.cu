// C ABI of the H100-native DSRG hot path (see include/dsrg_b200.h for the contract and the
// reference interfaces each entry point replaces).
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <initializer_list>
#include <map>
#include <mutex>
#include <utility>
#include <new>
#include <vector>

#include "common.cuh"

namespace dsrg {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int device_alloc(Engine *e, void **p, size_t bytes) {
    if (bytes == 0) bytes = 16;
    cudaError_t err = cudaMalloc(p, bytes);
    if (err != cudaSuccess) {
        set_error("cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(err));
        *p = nullptr;
        return DSRG_E_NOMEM;
    }
    e->bytes += bytes;
    return DSRG_OK;
}

// elevation scale factors exactly as the reference computes them (permutohedral.cpp:179-182):
// float inv_std_dev = sqrt(2/3)*(d+1); scale[i] = float(1.0/sqrt((i+2)*(i+1)) * inv_std_dev)
static void lattice_scales(Lattice &L) {
    const float inv_std_dev = (float)(sqrt(2.0 / 3.0) * (L.d + 1));
    for (int i = 0; i < L.d; i++)
        L.scale[i] = (float)(1.0 / sqrt((double)((i + 2) * (i + 1))) * (double)inv_std_dev);
}

// conservative host-side bound on |lattice key| so that range problems surface as an error code
// before anything is launched (the kernels keep a device-side flag as a second line of defence)
static bool key_range_ok(const Lattice &L, int W, int H) {
    double fmax[5] = {(W - 1) / (double)L.sigma[0], (H - 1) / (double)L.sigma[1], 0, 0, 0};
    for (int i = 2; i < L.d; i++) fmax[i] = 255.0 / (double)L.sigma[i];
    double sum = 0, big = 0;
    for (int i = 0; i < L.d; i++) {
        double cf = fabs(fmax[i]) * L.scale[i];
        sum += cf;
        if ((i + 1) * cf > big) big = (i + 1) * cf;
    }
    const double bound = sum + big + 3.0 * (L.d + 1) + 2;
    const int bits = (L.d == 2) ? 16 : 12;
    return bound < (double)((1 << (bits - 1)) - 1) && isfinite(bound);
}

// shape-dependent strides of a lattice family; every one of them grows with N, so buffers sized for
// the engine's capacity shape hold any smaller shape (dsrg_engine_set_size)
static void lattice_shape(Engine *e, Lattice &L) {
    L.N = e->N;
    L.P = (4 - (e->N % 4)) % 4;
    L.capv = (L.N + L.P) * (L.d + 1);
    L.cap = 2 * L.capv;
    L.rows_cap = (long long)e->maxB * (L.capv + 1);
    L.nbr_stride = L.shared ? (long long)L.capv + 1 : L.rows_cap;
}

static void engine_shape(Engine *e, int H, int W) {
    e->H = H;
    e->W = W;
    e->N = H * W;
    e->tiles_x = (W + kTileW - 1) / kTileW;
    e->tile_w = (W + e->tiles_x - 1) / e->tiles_x;  // e.g. W=321: 11 tiles of 30 instead of 10 x 32 + a 1-pixel sliver
    e->tiles_y = (H + kTileH - 1) / kTileH;
    e->ntiles = e->tiles_x * e->tiles_y;
    lattice_shape(e, e->sp);
    lattice_shape(e, e->bi);
    e->sp_valid = false;
}

// The renumbering key of an incidence, pos * (d+1) + r (lattice.cu: k_lattice_insert), is an int below kNoKey.  pos
// runs to ntiles * kTileThreads (the phantom lanes' position), so the bilateral lattice's largest key is
// ntiles * kTileThreads * 6 + 5.  Narrow images have few pixels per tile (one column: 8 of 256), and from
// 11 140 945 x 1 on the key would reach kNoKey.  set_size keeps the tile count at or below the capacity's.
static bool renum_keys_fit(int H, int W) {
    const long long tiles_x = (W + kTileW - 1) / kTileW, tiles_y = (H + kTileH - 1) / kTileH;
    return tiles_x * tiles_y * kTileThreads * 6 + 5 < (long long)kNoKey;
}

static int lattice_alloc(Engine *e, Lattice &L, int d, int shared) {
    L.d = d;
    L.shared = shared;
    L.nimg = shared ? 1 : e->maxB;
    lattice_shape(e, L);
    const size_t n = (size_t)L.nimg;
    int rc = 0;
    rc |= dalloc(e, &L.off, n * (d + 1) * L.N);
    rc |= dalloc(e, &L.bary, n * (d + 1) * L.N);
    rc |= dalloc(e, &L.norm, n * L.N);
    rc |= dalloc(e, &L.hkeys, n * L.cap);
    rc |= dalloc(e, &L.hval, n * L.cap);
    rc |= dalloc(e, &L.vslot, n * L.capv);
    rc |= dalloc(e, &L.vcount, n);
    rc |= dalloc(e, &L.aslot, n * L.capv);
    rc |= dalloc(e, &L.vkey, n * L.capv);
    L.slots_alloc = (long long)n * L.cap;
    L.verts_alloc = (long long)n * L.capv;
    const long long rn_words = renum_words(e->ntiles, d + 1);  // the capacity shape has the most tiles
    rc |= dalloc(e, &L.rn_words, n * rn_words);
    rc |= dalloc(e, &L.rn_chunk, n * (rn_words / kRenumChunk));
    rc |= dalloc(e, &L.rowbase, (size_t)e->maxB + 1);
    rc |= dalloc(e, &L.nbr, (size_t)(d + 1) * L.nbr_stride);
    L.maxloc = (d == 2) ? kMaxLocSp : kMaxLocHy;
    const size_t nt = n * e->ntiles;
    rc |= dalloc(e, &L.tl_nloc, nt);
    rc |= dalloc(e, &L.tl_hy, nt);
    // every segment is padded to an even entry count; a tile's block starts on 16 bytes (8 entries)
    L.entcap = (kTileThreads * (d + 1) + L.maxloc + 7) & ~7;
    rc |= dalloc(e, &L.tl_hdr, nt * L.maxloc);
    rc |= dalloc(e, &L.tl_pack, nt * L.entcap);
    rc |= dalloc(e, &L.tl_loc, n * (d + 1) * L.N);
    rc |= dalloc(e, &L.wn, n * (d + 1) * L.N);
    rc |= dalloc(e, &L.tl_w, nt * (d + 1) * kTileThreads);
    rc |= dalloc(e, &L.tl_li, nt * (d + 1) * kTileThreads);
    if (rc) return DSRG_E_NOMEM;
    if (cudaMemset(L.hkeys, 0xFF, sizeof(uint64_t) * n * L.cap) != cudaSuccess) return DSRG_E_CUDA;
    if (cudaMemset(L.tl_hy, 0, nt) != cudaSuccess) return DSRG_E_CUDA;
    if (cudaMemset(L.hval, 0xFF, sizeof(int32_t) * n * L.cap) != cudaSuccess) return DSRG_E_CUDA;
    if (cudaMemset(L.vkey, 0x7F, sizeof(int32_t) * n * L.capv) != cudaSuccess) return DSRG_E_CUDA;  // kNoKey
    return DSRG_OK;
}

static void lattice_free(Lattice &L) {
    cudaFree(L.off);
    cudaFree(L.bary);
    cudaFree(L.norm);
    cudaFree(L.hkeys);
    cudaFree(L.hval);
    cudaFree(L.vslot);
    cudaFree(L.vcount);
    cudaFree(L.aslot);
    cudaFree(L.vkey);
    cudaFree(L.rn_words);
    cudaFree(L.rn_chunk);
    cudaFree(L.rowbase);
    cudaFree(L.nbr);
    cudaFree(L.tl_nloc);
    cudaFree(L.tl_hy);
    cudaFree(L.tl_hdr);
    cudaFree(L.tl_pack);
    cudaFree(L.tl_loc);
    cudaFree(L.wn);
    cudaFree(L.tl_w);
    cudaFree(L.tl_li);
}

int check_device_flag(Engine *e, cudaStream_t s) {
    int flag = 0;
    DSRG_CUDA_TRY(cudaMemcpyAsync(&flag, e->dev_err, sizeof(int), cudaMemcpyDeviceToHost, s));
    DSRG_CUDA_TRY(cudaStreamSynchronize(s));
    if (flag != 0) {
        cudaMemsetAsync(e->dev_err, 0, sizeof(int), s);
        set_error("lattice coordinates exceed the packed-key range (sigma too small for this image size)");
        return flag;
    }
    return DSRG_OK;
}

// the shared spatial lattice, when crf_pass found it due
static int prepare_spatial(Engine *e, int B, const dsrg_crf_params &p, cudaStream_t s) {
    if (!e->sp_valid) {
        e->sp.sigma[0] = p.theta_gamma_x;
        e->sp.sigma[1] = p.theta_gamma_y;
        if (!key_range_ok(e->sp, e->W, e->H)) {
            set_error("spatial sigma (%g,%g) too small for %dx%d: lattice keys exceed 16 bits",
                      p.theta_gamma_x, p.theta_gamma_y, e->W, e->H);
            return DSRG_E_KEYRANGE;
        }
        int rc = lattice_build(e, e->sp, B, nullptr, s);
        if (rc) return rc;
    }
    return DSRG_OK;
}

// (re)build lattices for this call: spatial only when crf_pass found it due, bilateral always
static int prepare_lattices(Engine *e, int B, const uint8_t *image, const dsrg_crf_params &p,
                            cudaStream_t s) {
    if (!(p.theta_gamma_x > 0 && p.theta_gamma_y > 0 && p.theta_alpha_x > 0 && p.theta_alpha_y > 0 &&
          p.theta_beta_r > 0 && p.theta_beta_g > 0 && p.theta_beta_b > 0) || p.n_iters < 0) {
        set_error("CRF parameters must be positive");
        return DSRG_E_INVALID;
    }
    if (int rc = prepare_spatial(e, B, p, s)) return rc;
    e->bi.sigma[0] = p.theta_alpha_x;
    e->bi.sigma[1] = p.theta_alpha_y;
    e->bi.sigma[2] = p.theta_beta_r;
    e->bi.sigma[3] = p.theta_beta_g;
    e->bi.sigma[4] = p.theta_beta_b;
    if (!key_range_ok(e->bi, e->W, e->H)) {
        set_error("bilateral sigmas too small for %dx%d: lattice keys exceed the 12-bit packed range",
                  e->W, e->H);
        return DSRG_E_KEYRANGE;
    }
    return lattice_build(e, e->bi, B, image, s);
}

// A buffer that the entry points needing it allocate on their first call, so that an engine which never runs them
// keeps its footprint.  Sized for the engine's capacity (set_size never exceeds it).
struct LazyBuf {
    void **p;
    size_t bytes;
};
template <typename T>
static LazyBuf lazy(T *&p, size_t count) {
    return {(void **)&p, count * sizeof(T)};
}

// Allocates each buffer of `bufs` that is still NULL, so a call after a failed one allocates only what is missing.  The
// call may sit inside a caller's stream capture, where an allocation is allowed in relaxed mode only.
static int lazy_alloc(Engine *e, std::initializer_list<LazyBuf> bufs) {
    bool missing = false;
    for (const LazyBuf &b : bufs) missing |= *b.p == nullptr;
    if (!missing) return DSRG_OK;
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    DSRG_CUDA_TRY(cudaThreadExchangeStreamCaptureMode(&mode));
    int rc = DSRG_OK;
    for (const LazyBuf &b : bufs)
        if (!*b.p && device_alloc(e, b.p, b.bytes)) rc = DSRG_E_NOMEM;
    DSRG_CUDA_TRY(cudaThreadExchangeStreamCaptureMode(&mode));
    return rc;
}

// the feature passes' per-image key-range flags
int ensure_feat(Engine *e) { return lazy_alloc(e, {lazy(e->feat_bad, e->maxB)}); }

// the compatibility backward's per-tile partials, B * ntiles * 2 * M^2 floats
static int ensure_compat_part(Engine *e) {
    const size_t tiles = (size_t)((e->Wcap + kTileW - 1) / kTileW) * ((e->Hcap + kTileH - 1) / kTileH);
    return lazy_alloc(e, {lazy(e->compat_part, (size_t)e->maxB * tiles * 2 * e->M * e->M)});
}

// the kernel-bandwidth backward's buffers: g_t and c per pixel, the per-block sums and two value buffers per lattice
static int ensure_kgrad(Engine *e) {
    const size_t sp = (size_t)e->sp.rows_cap * e->MP, bi = (size_t)e->bi.rows_cap * e->MP;
    return lazy_alloc(e, {lazy(e->kg_g, (size_t)e->maxB * e->M * e->Ncap),
                          lazy(e->kg_csum, (size_t)2 * e->maxB * e->Ncap),
                          lazy(e->kg_part, (size_t)e->maxB * ((e->Ncap + kThreads - 1) / kThreads) * 8),
                          lazy(e->kg_sp[0], sp), lazy(e->kg_bi[0], bi), lazy(e->kg_sp[1], sp), lazy(e->kg_bi[1], bi)});
}

// the label-chunked backward's buffers: the Potts partials, and for the matrices G and the outer-product partials
static int ensure_wide(Engine *e, bool compat) {
    const LazyBuf ppart = lazy(e->wide_ppart, (size_t)e->maxB * (e->MP / 4) * ((e->Ncap + kThreads - 1) / kThreads));
    if (!compat) return lazy_alloc(e, {ppart});
    return lazy_alloc(e, {ppart, lazy(e->wide_g, (size_t)e->maxB * e->M * e->Ncap),
                          lazy(e->wide_cpart, (size_t)e->maxB * kWideChunks * 2 * e->M * e->M)});
}

// The label-chunked kernel-bandwidth and feature backward's buffers: c per pixel [2][maxB][N] and the per-block sums,
// as ensure_kgrad, and the normalisation term's two value buffers per lattice at 4 floats per row.  g_t stays in e->Q0
// and Vy in the mean-field buffers, so nothing here grows with the label count.
static int ensure_kgrad_wide(Engine *e) {
    const size_t sp = (size_t)e->sp.rows_cap * 4, bi = (size_t)e->bi.rows_cap * 4;
    return lazy_alloc(e, {lazy(e->kg_csum, (size_t)2 * e->maxB * e->Ncap),
                          lazy(e->kg_part, (size_t)e->maxB * ((e->Ncap + kThreads - 1) / kThreads) * 8),
                          lazy(e->kg_sp[0], sp), lazy(e->kg_bi[0], bi), lazy(e->kg_sp[1], sp), lazy(e->kg_bi[1], bi)});
}

// the energy's per-block sums, and with features the per-image flags
static int ensure_energy(Engine *e, bool feat) {
    if (feat)
        if (int rc = ensure_feat(e)) return rc;
    return lazy_alloc(e, {lazy(e->en_part, (size_t)e->maxB * ((e->Ncap + kThreads - 1) / kThreads) * 4)});
}

// prepare_lattices with caller-given bilateral features ([B][5][N]): the bilateral sigmas of `p` are not used, and the
// key range is checked per image on the device (e->feat_bad, which ensure_feat allocates)
static int prepare_lattices_feat(Engine *e, int B, const float *feat, const dsrg_crf_params &p, cudaStream_t s) {
    if (!(p.theta_gamma_x > 0 && p.theta_gamma_y > 0) || p.n_iters < 0) {
        set_error("CRF parameters must be positive");
        return DSRG_E_INVALID;
    }
    if (int rc = prepare_spatial(e, B, p, s)) return rc;
    for (int i = 0; i < 5; i++) e->bi.sigma[i] = 1.0f;
    return lattice_build(e, e->bi, B, nullptr, s, feat, e->feat_bad);
}

// the lattices of the image, or of caller-given bilateral features
static int prepare_lattices_for(Engine *e, int B, const uint8_t *image, const float *features,
                                const dsrg_crf_params &p, cudaStream_t s) {
    return features ? prepare_lattices_feat(e, B, features, p, s) : prepare_lattices(e, B, image, p, s);
}

// The feature passes' NaN policy: every value of a given output becomes NaN in the images whose feature lattice left
// the packed key range (e->feat_bad).  An output holds per_image floats per image, `reps` times over ([reps][B]...).
struct NanOut {
    float *p;
    long long per_image;
    int reps = 1;
};
static int nan_flagged_outputs(Engine *e, int B, std::initializer_list<NanOut> outs, cudaStream_t s,
                               int tag = T_FGRAD) {
    for (const NanOut &o : outs)
        if (o.p) nan_images(e, e->feat_bad, o.p, B, o.per_image, o.reps, s, tag);
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

int check_batch(Engine *e, int B) {
    if (!e) {
        set_error("engine is NULL");
        return DSRG_E_INVALID;
    }
    if (B < 1 || B > e->maxB) {
        set_error("batch %d outside [1, %d]", B, e->maxB);
        return DSRG_E_INVALID;
    }
    int cur = -1;  // the entry point's DeviceScope selected the engine's device
    if (cudaGetDevice(&cur) != cudaSuccess || cur != e->device) DSRG_CUDA_TRY(cudaSetDevice(e->device));
    return DSRG_OK;
}

bool crf_pass_begin(Engine *e, const dsrg_crf_params &p) {
    if (e->sp_valid && e->sp.sigma[0] == p.theta_gamma_x && e->sp.sigma[1] == p.theta_gamma_y) return false;
    e->sp_valid = false;  // prepare_lattices rebuilds it, in the pass and so in its graph
    return true;
}

void crf_pass_end(Engine *e, const dsrg_crf_params &p, int B, int rc) {
    if (rc != DSRG_OK) {
        e->last_crf_B = 0;
        return;
    }
    e->sp.sigma[0] = p.theta_gamma_x;
    e->sp.sigma[1] = p.theta_gamma_y;
    e->sp_valid = true;
    e->last_crf_B = B;
}

int crf_core(Engine *e, int B, const float *unary, int layout, bool clamp, float *unary_rw, const uint8_t *image,
             const dsrg_crf_params *p, cudaStream_t s, const LearnedCrf *lc) {
    if (layout != DSRG_LAYOUT_NHWC && layout != DSRG_LAYOUT_NCHW) {
        set_error("bad layout %d", layout);
        return DSRG_E_INVALID;
    }
    const float *feat = lc ? lc->features : nullptr;
    int rc = prepare_lattices_for(e, B, image, feat, *p, s);
    if (rc) return rc;
    if (!lc) return meanfield_run(e, B, unary, layout, clamp, unary_rw, *p, s);
    rc = meanfield_run(e, B, unary, layout, clamp, unary_rw, *p, s, lc->compat);
    if (rc || !feat) return rc;
    return nan_flagged_outputs(e, B, {{e->Q0, (long long)e->M * e->N}}, s);   // the training forward's policy
}

static int crf_batch_pass(Engine *e, int B, const float *unary, int unary_layout, const uint8_t *image,
                          const dsrg_crf_params *params, float *out, int out_layout, cudaStream_t s) {
    GraphKey args;
    args.add(unary).add(unary_layout).add(image).add(out).add(out_layout);
    return crf_pass(e, s, PassKind::crf, B, params, args, [&]() {
        int r = crf_core(e, B, unary, unary_layout, false, nullptr, image, params, s);
        if (r) return r;
        return meanfield_export(e, B, out, out_layout, s);
    });
}

static int crflayer_pass(Engine *e, int B, float *probs, const uint8_t *image, const dsrg_crf_params *params,
                         float *log_out, float *result, cudaStream_t s) {
    GraphKey args;
    args.add(probs).add(image).add(log_out).add(result);
    return crf_pass(e, s, PassKind::crflayer, B, params, args, [&]() {
        int r = crf_core(e, B, probs, DSRG_LAYOUT_NCHW, true, probs, image, params, s);
        if (r) return r;
        return meanfield_export_renorm(e, B, result, log_out, s);
    });
}

// the full pass; cues / seeds as float planes or (host pipeline, wire.cu) in the 1-bit wire format
int dsrg_forward_core(Engine *e, int B, const float *labels, float *probs, const float *cues, const uint32_t *cue_bits,
                      const uint8_t *image, const dsrg_crf_params *params, double th1, double th2, float *seeds_out,
                      uint32_t *seed_bits, float *crf_out, cudaStream_t s) {
    GraphKey args;
    args.add(labels).add(probs).add(cues).add(cue_bits).add(image).add(th1).add(th2).add(seeds_out).add(seed_bits).add(crf_out);
    return crf_pass(e, s, PassKind::forward, B, params, args, [&]() {
        // refinement (pylayers.py:310-331): in-place clamp, unary = probs (NCHW), CRF
        int r = crf_core(e, B, probs, DSRG_LAYOUT_NCHW, true, probs, image, params, s);
        if (r) return r;
        if (crf_out && (r = meanfield_export(e, B, crf_out, DSRG_LAYOUT_NCHW, s))) return r;
        // SRG on the raw marginals with the float64 clamp + renormalisation fused in (renorm = 1)
        return srg_run(e, B, labels, e->Q0, cues, th1, th2, 1, seeds_out, nullptr, s, cue_bits, seed_bits);
    });
}

int ensure_staging(Engine *e) {
    if (e->st_unary) return DSRG_OK;
    const size_t n = (size_t)e->maxB * e->M * e->Ncap;
    int rc = 0;
    rc |= dalloc(e, &e->st_unary, n);
    rc |= dalloc(e, &e->st_out, n);
    rc |= dalloc(e, &e->st_cues, n);
    rc |= dalloc(e, &e->st_labels, (size_t)e->maxB * e->M);
    rc |= dalloc(e, &e->st_image, (size_t)e->maxB * e->Ncap * 3);
    rc |= dalloc(e, &e->st_lmap, (size_t)e->maxB * e->Ncap);
    rc |= dalloc(e, &e->st_sel, (size_t)e->M);
    return rc ? DSRG_E_NOMEM : DSRG_OK;
}

int grow_staging(Engine *e, void **buf, size_t *cap_bytes, size_t bytes) {
    if (bytes <= *cap_bytes) return DSRG_OK;
    cudaFree(*buf);  // synchronises with anything still reading it
    *buf = nullptr;
    *cap_bytes = 0;
    if (int rc = device_alloc(e, buf, bytes)) return rc;
    *cap_bytes = bytes;
    return DSRG_OK;
}

static int no_engine() {
    set_error("engine is NULL");
    return DSRG_E_INVALID;
}

// the *_last_* entry points read what the engine's last mean-field pass left behind
static int last_crf_held(const Engine *e, int B) {
    if (e->last_crf_B == B) return DSRG_OK;
    set_error("no mean-field result for a batch of %d is held by this engine (last: %d)", B, e->last_crf_B);
    return DSRG_E_STATE;
}

static bool layout_ok(int layout) { return layout == DSRG_LAYOUT_NHWC || layout == DSRG_LAYOUT_NCHW; }

}  // namespace dsrg

using namespace dsrg;

extern "C" {

int dsrg_version(void) { return 119; }

const char *dsrg_last_error(void) { return g_err; }

int dsrg_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

int dsrg_current_device(void) {
    // the device the drop-ins create their engines on: DSRG_B200_DEVICE if set, else the calling thread's
    // current CUDA device (what caffe.set_device / torch.cuda.set_device selected), else LOCAL_RANK
    if (const char *ev = getenv("DSRG_B200_DEVICE")) return atoi(ev);
    int dev = -1;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    return dev;
}

void *dsrg_host_alloc(size_t bytes) {
    void *p = nullptr;
    // on the NUMA node of the calling thread's current device when several ranks share the host (numa.cu)
    if (numa_host_alloc(&p, bytes ? bytes : 16, dsrg_current_device()) != cudaSuccess) {
        set_error("cudaHostAlloc(%zu) failed", bytes);
        cudaGetLastError();
        return nullptr;
    }
    return p;
}

void dsrg_host_free(void *p) {
    if (p) cudaFreeHost(p);
}

int dsrg_host_register(void *p, size_t bytes) {
    if (!p || !bytes) return DSRG_E_INVALID;
    if (cudaHostRegister(p, bytes, cudaHostRegisterDefault) != cudaSuccess) {
        cudaGetLastError();
        set_error("cudaHostRegister(%zu bytes) failed", bytes);
        return DSRG_E_CUDA;
    }
    return DSRG_OK;
}

int dsrg_host_unregister(void *p) {
    if (!p) return DSRG_E_INVALID;
    if (cudaHostUnregister(p) != cudaSuccess) {
        cudaGetLastError();
        return DSRG_E_CUDA;
    }
    return DSRG_OK;
}

void dsrg_crf_params_default(dsrg_crf_params *p, float scale_factor, float color_factor, int maxiter) {
    // CRF/krahenbuhl2013/CRF.py:31-32
    p->w1 = 10.0f;
    p->theta_alpha_x = p->theta_alpha_y = (float)(80.0 / (double)scale_factor);
    p->theta_beta_r = p->theta_beta_g = p->theta_beta_b = color_factor;
    p->w2 = 3.0f;
    p->theta_gamma_x = p->theta_gamma_y = (float)(3.0 / (double)scale_factor);
    p->n_iters = maxiter;
}

dsrg_engine *dsrg_engine_create(int device, int max_batch, int H, int W, int M) {
    if (max_batch < 1 || H < 1 || W < 1 || M < 1 || M > DSRG_MAX_LABELS_WIDE ||
        (long long)H * W > (1ll << 24) || !renum_keys_fit(H, W)) {
        set_error("bad engine shape (max_batch=%d H=%d W=%d M=%d; M <= %d, H*W <= 2^24, lattice renumbering keys "
                  "below %d)", max_batch, H, W, M, DSRG_MAX_LABELS_WIDE, kNoKey);
        return nullptr;
    }
    int ndev = 0;
    if (device < 0) device = dsrg_current_device();  // -1: the calling thread's current device
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        set_error("no usable CUDA device %d (visible devices: %d): this library has no CPU fallback",
                  device, ndev);
        return nullptr;
    }
    cudaDeviceProp prop;
    Engine probe;
    probe.device = device;
    DeviceScope dev_scope(&probe);  // creation, too, leaves the caller's current device as it found it
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) {
        set_error("cannot select device %d", device);
        return nullptr;
    }
    if (prop.major != 9 || prop.minor != 0) {
        set_error("device %d is sm_%d%d; this build contains sm_90a code only", device, prop.major,
                  prop.minor);
        return nullptr;
    }
    Engine *e = new (std::nothrow) Engine();
    if (!e) return nullptr;
    e->device = device;
    if (numa_wanted()) {  // several ranks on this host: keep this rank's host side next to its GPU
        e->numa_node = numa_node_of_device(device);
        numa_bind_thread(e->numa_node);
    }
    e->maxB = max_batch;
    e->M = M;
    e->MP = (M + 3) / 4 * 4;
    e->sm_count = prop.multiProcessorCount;
    e->sp.d = 2;
    e->sp.shared = 1;
    e->bi.d = 5;
    e->Hcap = H;
    e->Wcap = W;
    e->Ncap = H * W;
    engine_shape(e, H, W);
    int rc = 0;
    rc |= lattice_alloc(e, e->sp, 2, 1);
    rc |= lattice_alloc(e, e->bi, 5, 0);
    lattice_scales(e->sp);
    lattice_scales(e->bi);
    const size_t n = (size_t)max_batch * M * e->N;
    rc |= dalloc(e, &e->U, n);
    rc |= dalloc(e, &e->Q0, n);
    rc |= dalloc(e, &e->spA, (size_t)e->sp.rows_cap * e->MP);
    rc |= dalloc(e, &e->spB, (size_t)e->sp.rows_cap * e->MP);
    rc |= dalloc(e, &e->spC, (size_t)e->sp.rows_cap * e->MP);
    rc |= dalloc(e, &e->biC, (size_t)e->bi.rows_cap * e->MP);
    rc |= dalloc(e, &e->biA, (size_t)e->bi.rows_cap * e->MP);
    rc |= dalloc(e, &e->biB, (size_t)e->bi.rows_cap * e->MP);
    rc |= dalloc(e, &e->nvA, (size_t)e->bi.rows_cap);
    rc |= dalloc(e, &e->nvB, (size_t)e->bi.rows_cap);
    const size_t bn = (size_t)max_batch * e->N;
    rc |= dalloc(e, &e->lmap, bn);
    rc |= dalloc(e, &e->lflag, bn);
    rc |= dalloc(e, &e->parent, bn);
    rc |= dalloc(e, &e->hc, bn);
    rc |= dalloc(e, &e->loss_acc, (size_t)max_batch * 4);
    e->sec_wcap = e->Ncap < DSRG_GWRP_MAX_PLANE ? e->Ncap : DSRG_GWRP_MAX_PLANE;
    rc |= dalloc(e, &e->sec_rec, (size_t)max_batch * M);
    rc |= dalloc(e, &e->sec_img, (size_t)max_batch * 3);
    rc |= dalloc(e, &e->sec_part, (size_t)max_batch * kSecPlainChunks);
    rc |= dalloc(e, &e->sec_w, (size_t)2 * e->sec_wcap);
    rc |= dalloc(e, &e->dev_err, 1);
    rc |= dalloc(e, &e->hy_list, (size_t)max_batch * e->ntiles);
    rc |= dalloc(e, &e->potts_part, (size_t)max_batch * e->ntiles);
    rc |= dalloc(e, &e->hy_count, 1);
    if (!rc && cudaMemset(e->hy_count, 0, sizeof(int)) != cudaSuccess) rc = DSRG_E_CUDA;
    if (!rc && cudaMemset(e->dev_err, 0, sizeof(int)) != cudaSuccess) rc = DSRG_E_CUDA;
    if (!rc && cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking) != cudaSuccess) rc = DSRG_E_CUDA;
    if (!rc && cudaStreamCreateWithFlags(&e->in_stream, cudaStreamNonBlocking) != cudaSuccess) rc = DSRG_E_CUDA;
    if (!rc && cudaEventCreateWithFlags(&e->order_event, cudaEventDisableTiming) != cudaSuccess) rc = DSRG_E_CUDA;
    if (const char *ev = getenv("DSRG_B200_WIRE")) e->wire_compress = atoi(ev) != 0;
    if (const char *ev = getenv("DSRG_B200_GRAPHS")) e->use_graphs = atoi(ev) != 0;
    if (const char *ev = getenv("DSRG_B200_HOST_CHUNK")) e->host_chunk = atoi(ev) > 0 ? atoi(ev) : e->host_chunk;
    if (!rc && cudaStreamCreateWithFlags(&e->out_stream, cudaStreamNonBlocking) != cudaSuccess) rc = DSRG_E_CUDA;
    if (rc) {
        dsrg_engine_destroy((dsrg_engine *)e);
        return nullptr;
    }
    return (dsrg_engine *)e;
}

void dsrg_engine_destroy(dsrg_engine *h) {
    Engine *e = (Engine *)h;
    if (!e) return;
    DeviceScope dev_scope(e);
    cudaDeviceSynchronize();
    graph_clear(e);
    lattice_free(e->sp);
    lattice_free(e->bi);
    void *ptrs[] = {e->U, e->Q0, e->spA, e->spB, e->spC, e->biA, e->biB, e->biC, e->nvA, e->nvB, e->lmap,
                    e->lflag, e->parent, e->hc, e->loss_acc, e->sec_rec, e->sec_img, e->sec_part, e->sec_w, e->dev_err,
                    e->hy_list, e->hy_count, e->potts_part, e->compat_part, e->kg_g, e->kg_csum, e->kg_part, e->kg_sp[0],
                    e->kg_sp[1], e->kg_bi[0], e->kg_bi[1], e->feat_bad, e->wide_ppart, e->wide_g, e->wide_cpart, e->en_part, e->st_unary, e->st_out, e->st_cues, e->st_labels, e->st_image, e->st_lmap, e->st_raw, e->st_idx,
                    e->st_prep, e->st_sel};
    for (void *p : ptrs) cudaFree(p);
    if (e->own_stream) cudaStreamDestroy(e->own_stream);
    if (e->in_stream) cudaStreamDestroy(e->in_stream);
    if (e->order_event) cudaEventDestroy(e->order_event);
    if (e->out_stream) cudaStreamDestroy(e->out_stream);
    for (auto ev : e->pipe_events) cudaEventDestroy(ev);
    wire_free(e);
    for (auto &r : e->prof_recs) {
        cudaEventDestroy(r.a);
        cudaEventDestroy(r.b);
    }
    for (auto ev : e->prof_pool) cudaEventDestroy(ev);
    delete e;
}

size_t dsrg_engine_device_bytes(const dsrg_engine *h) { return h ? ((const Engine *)h)->bytes : 0; }

// wait: for the work already queued on any stream.  Queued launches keep the old strides in their arguments, so the
// wait is only needed for work the engine cannot order: dsrg_engine_set_size_ordered skips it.
static int set_size(Engine *e, int H, int W, bool wait) {
    if (!e) return no_engine();
    if (H < 1 || W < 1 || H > e->Hcap || W > e->Wcap) {
        set_error("size %dx%d outside the engine's capacity %dx%d", H, W, e->Hcap, e->Wcap);
        return DSRG_E_INVALID;
    }
    if (H == e->H && W == e->W) return DSRG_OK;
    if (wait) {
        DeviceScope dev_scope(e);
        DSRG_CUDA_TRY(cudaDeviceSynchronize());
    }
    engine_shape(e, H, W);
    e->last_crf_B = 0;
    // cached graphs stay: they are keyed by the shape (every stride is a function of it and of the capacity the
    // buffers were sized for), so a per-image caller that meets a size again replays that size's graph
    return DSRG_OK;
}

int dsrg_engine_set_size(dsrg_engine *h, int H, int W) { return set_size((Engine *)h, H, W, true); }

// Every entry point orders its pass after the engine's previous one (StreamScope: the same stream, or a wait for the
// order event on another), so between passes issued through the entry points the re-shape needs no wait
int dsrg_engine_set_size_ordered(dsrg_engine *h, int H, int W) { return set_size((Engine *)h, H, W, false); }

int dsrg_engine_get_size(const dsrg_engine *h, int *H, int *W, int *Hcap, int *Wcap) {
    const Engine *e = (const Engine *)h;
    if (!e) return no_engine();
    if (H) *H = e->H;
    if (W) *W = e->W;
    if (Hcap) *Hcap = e->Hcap;
    if (Wcap) *Wcap = e->Wcap;
    return DSRG_OK;
}

long long dsrg_engine_take_launch_count(dsrg_engine *h) {
    Engine *e = (Engine *)h;
    if (!e) return 0;
    long long n = e->launches;
    e->launches = 0;
    return n;
}

static const char *kTagNames[T_COUNT] = {
    "lattice_insert", "lattice_misc", "lattice_norm", "mf_init", "mf_zero", "mf_blur_spatial",
    "mf_blur_bilateral", "mf_tile", "mf_export", "srg_label", "srg_merge", "srg_flag", "srg_emit",
    "seedloss", "wire_bits", "prepare_image", "postprocess", "annotation", "mf_tile_hybrid",
    "kernel_grad", "feature_grad", "wide_grad", "crf_energy"};

int dsrg_profile_tag_count(void) { return T_COUNT; }

const char *dsrg_profile_tag_name(int tag) { return (tag >= 0 && tag < T_COUNT) ? kTagNames[tag] : ""; }

int dsrg_engine_set_host_chunk(dsrg_engine *h, int images) {
    Engine *e = (Engine *)h;
    if (!e) return no_engine();
    if (images < 0) return DSRG_E_INVALID;
    e->host_chunk = images;
    return DSRG_OK;
}

int dsrg_engine_set_graphs(dsrg_engine *h, int enable) {
    Engine *e = (Engine *)h;
    if (!e) return no_engine();
    e->use_graphs = enable != 0;
    if (!enable) {
        DeviceScope dev_scope(e);
        cudaDeviceSynchronize();
        graph_clear(e);
    }
    return DSRG_OK;
}

long long dsrg_engine_graph_replays(const dsrg_engine *h) { return h ? ((const Engine *)h)->graph_replays : 0; }
long long dsrg_engine_hybrid_tiles(dsrg_engine *h) {
    Engine *e = (Engine *)h;
    if (!e) return -1;
    DeviceScope dev_scope(e);
    int n = 0;
    if (cudaDeviceSynchronize() != cudaSuccess ||
        cudaMemcpy(&n, e->hy_count, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) {
        set_error("reading the hybrid-tile count failed: %s", cudaGetErrorString(cudaGetLastError()));
        return -1;
    }
    return n;
}

int dsrg_engine_profile(dsrg_engine *h, int enable) {
    Engine *e = (Engine *)h;
    if (!e) return no_engine();
    e->prof = enable != 0;
    return DSRG_OK;
}

int dsrg_engine_profile_read(dsrg_engine *h, float *ms_out, long long *count_out) {
    Engine *e = (Engine *)h;
    if (!e) return no_engine();
    if (!ms_out || !count_out) return DSRG_E_INVALID;
    DeviceScope dev_scope(e);
    DSRG_CUDA_TRY(cudaDeviceSynchronize());
    for (int t = 0; t < T_COUNT; t++) {
        ms_out[t] = 0.0f;
        count_out[t] = 0;
    }
    for (auto &r : e->prof_recs) {
        float ms = 0.0f;
        if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
            ms_out[r.tag] += ms;
            count_out[r.tag] += 1;
        }
        e->prof_pool.push_back(r.a);
        e->prof_pool.push_back(r.b);
    }
    e->prof_recs.clear();
    return DSRG_OK;
}

int dsrg_crf_batch_dev(dsrg_engine *h, int B, const float *unary, int unary_layout,
                       const uint8_t *image, const dsrg_crf_params *params, float *out,
                       int out_layout, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, unary && image && params && out && layout_ok(out_layout), [&](Engine *e) {
        return crf_batch_pass(e, B, unary, unary_layout, image, params, out, out_layout, s);
    });
}

// one training path per label count: these entry points run the fused kernels, the *_wide_dev pair the label-chunked
// ones above them
static int grad_labels_ok(const Engine *e) {
    if (e->MP <= DSRG_MAX_LABELS) return DSRG_OK;
    set_error("this CRF gradient supports at most %d labels (got %d); above 32 labels use "
              "dsrg_crf_forward_train_wide_dev / dsrg_crf_backward_wide_dev (or _wide_theta / _wide_feat)",
              DSRG_MAX_LABELS, e->M);
    return DSRG_E_INVALID;
}

static int wide_labels_ok(const Engine *e) {
    if (e->M > DSRG_MAX_LABELS) return DSRG_OK;
    set_error("the label-chunked CRF gradient takes more than %d labels (got %d); use the fused pair "
              "dsrg_crf_forward_train_dev / dsrg_crf_backward_dev (or its _compat twin)", DSRG_MAX_LABELS, e->M);
    return DSRG_E_INVALID;
}

static GraphKey train_key(const CrfTrainIo &io) {
    GraphKey args;
    args.add(io.unary).add(io.q_hist).add(io.grad_q).add(io.image).add(io.features).add(io.potts).add(io.compat)
        .add(io.q_out).add(io.grad_unary).add(io.grad_potts).add(io.grad_compat).add(io.grad_theta)
        .add(io.grad_features).add(io.grad_theta_sp);
    return args;
}

// What a pass that leaves no marginals in the engine notes: the *_last_* entry points refuse, and a feature pass's
// batch is the one dsrg_engine_feature_range_flags reports on
static int learned_pass_end(Engine *e, int B, const float *features, int rc) {
    e->last_crf_B = 0;
    if (features) e->feat_B = rc == DSRG_OK ? B : 0;
    return rc;
}

// The body of every training forward: Q_0..Q_T to io.q_out, on the fused kernels or (wide) the label-chunked ones
static int train_forward(dsrg_engine *h, int B, cudaStream_t s, bool args_ok, PassKind kind, bool wide,
                         const dsrg_crf_params *params, const CrfTrainIo &io) {
    return dev_call(h, B, s, args_ok, [&](Engine *e) {
        if (int rc = wide ? wide_labels_ok(e) : grad_labels_ok(e)) return rc;
        if (io.features)
            if (int rc = ensure_feat(e)) return rc;
        const int rc = crf_pass(e, s, kind, B, params, train_key(io), [&]() {
            int r = prepare_lattices_for(e, B, io.image, io.features, *params, s);
            if (!r) r = (wide ? meanfield_run_train_wide : meanfield_run_train)(e, B, io, *params, s);
            if (r || !io.features) return r;
            // every kept iterate
            return nan_flagged_outputs(e, B, {{io.q_out, (long long)e->M * e->N, params->n_iters + 1}}, s);
        });
        return learned_pass_end(e, B, io.features, rc);
    });
}

// The body of every training backward: the buffers its outputs need on their first call, then the gradients
static int train_backward(dsrg_engine *h, int B, cudaStream_t s, bool args_ok, PassKind kind, bool wide,
                          const dsrg_crf_params *params, const CrfTrainIo &io) {
    return dev_call(h, B, s, args_ok, [&](Engine *e) {
        if (int rc = wide ? wide_labels_ok(e) : grad_labels_ok(e)) return rc;
        int rc = wide ? ensure_wide(e, io.compat != nullptr) : io.compat ? ensure_compat_part(e) : DSRG_OK;
        if (!rc && (io.grad_theta || io.features)) rc = wide ? ensure_kgrad_wide(e) : ensure_kgrad(e);
        if (!rc && io.features) rc = ensure_feat(e);
        if (rc) return rc;
        rc = crf_pass(e, s, kind, B, params, train_key(io), [&]() {
            // the lattices are rebuilt: autograd may have run other passes on this engine since the forward
            int r = prepare_lattices_for(e, B, io.image, io.features, *params, s);
            if (!r) r = (wide ? meanfield_backward_wide : meanfield_backward)(e, B, io, *params, s);
            if (r || !io.features) return r;
            const long long M = e->M, N = e->N;
            return nan_flagged_outputs(e, B, {{io.grad_unary, M * N}, {io.grad_features, 5 * N}, {io.grad_potts, 2},
                                              {io.grad_compat, 2 * M * M}, {io.grad_theta_sp, 2}}, s);
        });
        return learned_pass_end(e, B, io.features, rc);
    });
}

int dsrg_crf_forward_train_dev(dsrg_engine *h, const float *unary, int B, const uint8_t *image,
                               const dsrg_crf_params *params, const float *potts, float *q_hist, void *stream) {
    return train_forward(h, B, (cudaStream_t)stream, unary && image && params && q_hist, PassKind::crf_train, false,
                         params, {.unary = unary, .image = image, .potts = potts, .q_out = q_hist});
}

int dsrg_crf_backward_dev(dsrg_engine *h, const float *q_hist, int B, const uint8_t *image,
                          const dsrg_crf_params *params, const float *potts, const float *grad_q, float *grad_unary,
                          float *grad_potts, void *stream) {
    return train_backward(h, B, (cudaStream_t)stream, q_hist && image && params && grad_q && grad_unary,
                          PassKind::crf_backward, false, params,
                          {.q_hist = q_hist, .grad_q = grad_q, .image = image, .potts = potts, .grad_unary = grad_unary,
                           .grad_potts = grad_potts});
}

int dsrg_crf_forward_train_compat_dev(dsrg_engine *h, const float *unary, int B, const uint8_t *image,
                                      const dsrg_crf_params *params, const float *compat, float *q_hist, void *stream) {
    return train_forward(h, B, (cudaStream_t)stream, unary && image && params && compat && q_hist,
                         PassKind::crf_train_compat, false, params,
                         {.unary = unary, .image = image, .compat = compat, .q_out = q_hist});
}

int dsrg_crf_backward_compat_dev(dsrg_engine *h, const float *q_hist, int B, const uint8_t *image,
                                 const dsrg_crf_params *params, const float *compat, const float *grad_q,
                                 float *grad_unary, float *grad_compat, void *stream) {
    return train_backward(h, B, (cudaStream_t)stream, q_hist && image && params && compat && grad_q && grad_unary,
                          PassKind::crf_backward_compat, false, params,
                          {.q_hist = q_hist, .grad_q = grad_q, .image = image, .compat = compat,
                           .grad_unary = grad_unary, .grad_compat = grad_compat});
}

int dsrg_crf_backward_theta_dev(dsrg_engine *h, const float *q_hist, int B, const uint8_t *image,
                                const dsrg_crf_params *params, const float *potts, const float *grad_q,
                                float *grad_unary, float *grad_potts, float *grad_theta, void *stream) {
    return train_backward(h, B, (cudaStream_t)stream,
                          q_hist && image && params && grad_q && grad_unary && grad_theta,
                          PassKind::crf_backward_theta, false, params,
                          {.q_hist = q_hist, .grad_q = grad_q, .image = image, .potts = potts,
                           .grad_unary = grad_unary, .grad_potts = grad_potts, .grad_theta = grad_theta});
}

int dsrg_crf_backward_compat_theta_dev(dsrg_engine *h, const float *q_hist, int B, const uint8_t *image,
                                       const dsrg_crf_params *params, const float *compat, const float *grad_q,
                                       float *grad_unary, float *grad_compat, float *grad_theta, void *stream) {
    return train_backward(h, B, (cudaStream_t)stream,
                          q_hist && image && params && compat && grad_q && grad_unary && grad_theta,
                          PassKind::crf_backward_compat_theta, false, params,
                          {.q_hist = q_hist, .grad_q = grad_q, .image = image, .compat = compat,
                           .grad_unary = grad_unary, .grad_compat = grad_compat, .grad_theta = grad_theta});
}

int dsrg_crf_forward_train_feat_dev(dsrg_engine *h, const float *unary, int B, const float *features,
                                    const dsrg_crf_params *params, const float *potts, const float *compat,
                                    float *q_hist, void *stream) {
    return train_forward(h, B, (cudaStream_t)stream, unary && features && params && q_hist && !(potts && compat),
                         PassKind::crf_train_feat, false, params,
                         {.unary = unary, .features = features, .potts = potts, .compat = compat, .q_out = q_hist});
}

int dsrg_crf_backward_feat_dev(dsrg_engine *h, const float *q_hist, int B, const float *features,
                               const dsrg_crf_params *params, const float *potts, const float *compat,
                               const float *grad_q, float *grad_unary, float *grad_features, float *grad_potts,
                               float *grad_compat, float *grad_theta_sp, void *stream) {
    const bool ok = q_hist && features && params && grad_q && grad_unary && grad_features && !(potts && compat) &&
                    !(grad_potts && compat) && !(grad_compat && !compat);
    return train_backward(h, B, (cudaStream_t)stream, ok, PassKind::crf_backward_feat, false, params,
                          {.q_hist = q_hist, .grad_q = grad_q, .features = features, .potts = potts, .compat = compat,
                           .grad_unary = grad_unary, .grad_potts = grad_potts, .grad_compat = grad_compat,
                           .grad_features = grad_features, .grad_theta_sp = grad_theta_sp});
}

int dsrg_engine_feature_range_flags(dsrg_engine *h, int B, int32_t *flags_out) {
    Engine *e = (Engine *)h;
    if (!e) return no_engine();
    if (!flags_out) return DSRG_E_INVALID;
    DeviceScope dev_scope(e);
    if (e->feat_B == 0 || B != e->feat_B) {
        set_error("the engine's last feature pass was not a batch of %d (last: %d)", B, e->feat_B);
        return DSRG_E_STATE;
    }
    DSRG_CUDA_TRY(cudaDeviceSynchronize());
    DSRG_CUDA_TRY(cudaMemcpy(flags_out, e->feat_bad, sizeof(int32_t) * B, cudaMemcpyDeviceToHost));
    return DSRG_OK;
}

int dsrg_crf_forward_train_wide_dev(dsrg_engine *h, const float *unary, int B, const uint8_t *image,
                                    const dsrg_crf_params *params, const float *potts, const float *compat,
                                    float *q_hist, void *stream) {
    return train_forward(h, B, (cudaStream_t)stream, unary && image && params && q_hist && !(potts && compat),
                         PassKind::crf_train_wide, true, params,
                         {.unary = unary, .image = image, .potts = potts, .compat = compat, .q_out = q_hist});
}

int dsrg_crf_backward_wide_dev(dsrg_engine *h, const float *q_hist, int B, const uint8_t *image,
                               const dsrg_crf_params *params, const float *potts, const float *compat,
                               const float *grad_q, float *grad_unary, float *grad_potts, float *grad_compat,
                               void *stream) {
    const bool ok = q_hist && image && params && grad_q && grad_unary && !(potts && compat) &&
                    !(grad_potts && compat) && !(grad_compat && !compat);
    return train_backward(h, B, (cudaStream_t)stream, ok, PassKind::crf_backward_wide, true, params,
                          {.q_hist = q_hist, .grad_q = grad_q, .image = image, .potts = potts, .compat = compat,
                           .grad_unary = grad_unary, .grad_potts = grad_potts, .grad_compat = grad_compat});
}

int dsrg_crf_backward_wide_theta_dev(dsrg_engine *h, const float *q_hist, int B, const uint8_t *image,
                                     const dsrg_crf_params *params, const float *potts, const float *compat,
                                     const float *grad_q, float *grad_unary, float *grad_potts, float *grad_compat,
                                     float *grad_theta, void *stream) {
    const bool ok = q_hist && image && params && grad_q && grad_unary && grad_theta && !(potts && compat) &&
                    !(grad_potts && compat) && !(grad_compat && !compat);
    return train_backward(h, B, (cudaStream_t)stream, ok, PassKind::crf_backward_wide_theta, true, params,
                          {.q_hist = q_hist, .grad_q = grad_q, .image = image, .potts = potts, .compat = compat,
                           .grad_unary = grad_unary, .grad_potts = grad_potts, .grad_compat = grad_compat,
                           .grad_theta = grad_theta});
}

int dsrg_crf_forward_train_wide_feat_dev(dsrg_engine *h, const float *unary, int B, const float *features,
                                         const dsrg_crf_params *params, const float *potts, const float *compat,
                                         float *q_hist, void *stream) {
    return train_forward(h, B, (cudaStream_t)stream, unary && features && params && q_hist && !(potts && compat),
                         PassKind::crf_train_wide_feat, true, params,
                         {.unary = unary, .features = features, .potts = potts, .compat = compat, .q_out = q_hist});
}

int dsrg_crf_backward_wide_feat_dev(dsrg_engine *h, const float *q_hist, int B, const float *features,
                                    const dsrg_crf_params *params, const float *potts, const float *compat,
                                    const float *grad_q, float *grad_unary, float *grad_features, float *grad_potts,
                                    float *grad_compat, float *grad_theta_sp, void *stream) {
    const bool ok = q_hist && features && params && grad_q && grad_unary && grad_features && !(potts && compat) &&
                    !(grad_potts && compat) && !(grad_compat && !compat);
    return train_backward(h, B, (cudaStream_t)stream, ok, PassKind::crf_backward_wide_feat, true, params,
                          {.q_hist = q_hist, .grad_q = grad_q, .features = features, .potts = potts, .compat = compat,
                           .grad_unary = grad_unary, .grad_potts = grad_potts, .grad_compat = grad_compat,
                           .grad_features = grad_features, .grad_theta_sp = grad_theta_sp});
}

// The body of the energy entry points: the lattices of the image or of the features, the energy (terms) or its
// gradient (grad_terms given) on the fused kernels or (wide) the label-chunked ones, and the feature passes' NaN policy
// for the outputs
static int energy_pass(Engine *e, int B, const float *q, const float *unary, const uint8_t *image, const float *features,
                       const dsrg_crf_params &p, const float *potts, const float *compat, float *terms,
                       const float *grad_terms, float *grad_q, float *grad_unary, bool wide, cudaStream_t s) {
    int r = prepare_lattices_for(e, B, image, features, p, s);
    if (!r)
        r = (wide ? meanfield_energy_wide : meanfield_energy)(e, B, q, unary, potts, compat, p, terms, grad_terms,
                                                                grad_q, grad_unary, s);
    if (r || !features) return r;
    const long long MN = (long long)e->M * e->N;
    return nan_flagged_outputs(e, B, {{terms, 4}, {grad_q, MN}, {grad_unary, MN}}, s, T_CRF_ENERGY);
}

// one energy path per label count, as for the training entry points
static int energy_labels_ok(const Engine *e, bool wide) {
    if (wide) {
        if (e->M > DSRG_MAX_LABELS) return DSRG_OK;
        set_error("the label-chunked CRF energy takes more than %d labels (got %d); use dsrg_crf_energy_dev / "
                  "dsrg_crf_energy_backward_dev", DSRG_MAX_LABELS, e->M);
        return DSRG_E_INVALID;
    }
    if (e->MP <= DSRG_MAX_LABELS) return DSRG_OK;
    set_error("the CRF energy supports at most %d labels (got %d)", DSRG_MAX_LABELS, e->M);
    return DSRG_E_INVALID;
}

static int energy_forward(dsrg_engine *h, const float *q, int B, const float *unary, const uint8_t *image,
                          const float *features, const dsrg_crf_params *params, const float *potts,
                          const float *compat, float *terms, void *stream, bool wide) {
    const cudaStream_t s = (cudaStream_t)stream;
    const bool ok = q && params && terms && (image != nullptr) != (features != nullptr) && !(potts && compat);
    return dev_call(h, B, s, ok, [&](Engine *e) {
        if (int rc = energy_labels_ok(e, wide)) return rc;
        if (int rc = ensure_energy(e, features != nullptr)) return rc;
        GraphKey args;
        args.add(q).add(unary).add(image).add(features).add(potts).add(compat).add(terms);
        const int rc = crf_pass(e, s, wide ? PassKind::crf_energy_wide : PassKind::crf_energy, B, params, args, [&]() {
            return energy_pass(e, B, q, unary, image, features, *params, potts, compat, terms, nullptr, nullptr,
                               nullptr, wide, s);
        });
        return learned_pass_end(e, B, features, rc);
    });
}

static int energy_backward(dsrg_engine *h, const float *q, int B, const float *unary, const uint8_t *image,
                           const float *features, const dsrg_crf_params *params, const float *potts,
                           const float *compat, const float *grad_terms, float *grad_q, float *grad_unary,
                           void *stream, bool wide) {
    const cudaStream_t s = (cudaStream_t)stream;
    const bool ok = q && params && grad_terms && grad_q && (image != nullptr) != (features != nullptr) &&
                    !(potts && compat);
    return dev_call(h, B, s, ok, [&](Engine *e) {
        if (int rc = energy_labels_ok(e, wide)) return rc;
        if (int rc = ensure_energy(e, features != nullptr)) return rc;
        GraphKey args;
        args.add(q).add(unary).add(image).add(features).add(potts).add(compat).add(grad_terms).add(grad_q)
            .add(grad_unary);
        const PassKind kind = wide ? PassKind::crf_energy_backward_wide : PassKind::crf_energy_backward;
        const int rc = crf_pass(e, s, kind, B, params, args, [&]() {
            return energy_pass(e, B, q, unary, image, features, *params, potts, compat, nullptr, grad_terms, grad_q,
                               grad_unary, wide, s);
        });
        return learned_pass_end(e, B, features, rc);
    });
}

int dsrg_crf_energy_dev(dsrg_engine *h, const float *q, int B, const float *unary, const uint8_t *image,
                        const float *features, const dsrg_crf_params *params, const float *potts, const float *compat,
                        float *terms, void *stream) {
    return energy_forward(h, q, B, unary, image, features, params, potts, compat, terms, stream, false);
}

int dsrg_crf_energy_backward_dev(dsrg_engine *h, const float *q, int B, const float *unary, const uint8_t *image,
                                 const float *features, const dsrg_crf_params *params, const float *potts,
                                 const float *compat, const float *grad_terms, float *grad_q, float *grad_unary,
                                 void *stream) {
    return energy_backward(h, q, B, unary, image, features, params, potts, compat, grad_terms, grad_q, grad_unary,
                           stream, false);
}

int dsrg_crf_energy_wide_dev(dsrg_engine *h, const float *q, int B, const float *unary, const uint8_t *image,
                             const float *features, const dsrg_crf_params *params, const float *potts,
                             const float *compat, float *terms, void *stream) {
    return energy_forward(h, q, B, unary, image, features, params, potts, compat, terms, stream, true);
}

int dsrg_crf_energy_backward_wide_dev(dsrg_engine *h, const float *q, int B, const float *unary, const uint8_t *image,
                                      const float *features, const dsrg_crf_params *params, const float *potts,
                                      const float *compat, const float *grad_terms, float *grad_q, float *grad_unary,
                                      void *stream) {
    return energy_backward(h, q, B, unary, image, features, params, potts, compat, grad_terms, grad_q, grad_unary,
                           stream, true);
}

int dsrg_crf_batch_learned_dev(dsrg_engine *h, const float *unary, int B, int unary_layout, const uint8_t *image,
                               const float *features, const dsrg_crf_params *params, const float *compat, float *out,
                               int out_layout, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    const bool ok = unary && params && out && layout_ok(unary_layout) && layout_ok(out_layout) &&
                    (image != nullptr) != (features != nullptr);
    return dev_call(h, B, s, ok, [&](Engine *e) {
        if (features)
            if (int rc = ensure_feat(e)) return rc;
        const LearnedCrf lc{features, compat};
        GraphKey args;
        args.add(unary).add(unary_layout).add(image).add(features).add(compat).add(out).add(out_layout);
        const int rc = crf_pass(e, s, PassKind::crf_learned, B, params, args, [&]() {
            int r = crf_core(e, B, unary, unary_layout, false, nullptr, image, params, s, &lc);
            if (r) return r;
            return meanfield_export(e, B, out, out_layout, s);
        });
        if (features) e->feat_B = rc == DSRG_OK ? B : 0;
        return rc;
    });
}

int dsrg_crf_map_batch_dev(dsrg_engine *h, int B, const float *unary, int unary_layout,
                           const uint8_t *image, const dsrg_crf_params *params, int32_t *labels_out,
                           void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, unary && image && params && labels_out, [&](Engine *e) {
        GraphKey args;
        args.add(unary).add(unary_layout).add(image).add(labels_out);
        return crf_pass(e, s, PassKind::crf_map, B, params, args, [&]() {
            int r = crf_core(e, B, unary, unary_layout, false, nullptr, image, params, s);
            if (r) return r;
            return meanfield_export_map(e, B, labels_out, s);
        });
    });
}

int dsrg_crf_batch_host(dsrg_engine *h, int B, const float *unary, int unary_layout,
                        const uint8_t *image, const dsrg_crf_params *params, float *out,
                        int out_layout) {
    return host_call(h, B, unary && image && params && out && layout_ok(out_layout), true, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, unary, n * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_image, image, (size_t)B * e->N * 3, cudaMemcpyHostToDevice, s));
        if (int rc = crf_batch_pass(e, B, e->st_unary, unary_layout, e->st_image, params, e->st_out, out_layout, s))
            return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(out, e->st_out, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}

int dsrg_srg_batch_dev(dsrg_engine *h, int B, const float *labels, const float *probs,
                       const float *cues, double th1, double th2, int renorm, float *seeds_out,
                       int32_t *label_map_out, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, labels && probs && cues && seeds_out, [&](Engine *e) {
        if (e->M > 255) {
            set_error("SRG supports at most 255 classes");
            return DSRG_E_INVALID;
        }
        return srg_run(e, B, labels, probs, cues, th1, th2, renorm, seeds_out, label_map_out, s);
    });
}

int dsrg_dsrg_forward_dev(dsrg_engine *h, int B, const float *labels, float *probs,
                          const float *cues, const uint8_t *image, const dsrg_crf_params *params,
                          double th1, double th2, float *seeds_out, float *crf_out, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, labels && probs && cues && image && params && seeds_out, [&](Engine *e) {
        return dsrg_forward_core(e, B, labels, probs, cues, nullptr, image, params, th1, th2, seeds_out, nullptr,
                                 crf_out, s);
    });
}

int dsrg_crflayer_forward_dev(dsrg_engine *h, int B, float *probs, const uint8_t *image,
                              const dsrg_crf_params *params, float *log_out, float *result,
                              void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, probs && image && params && log_out, [&](Engine *e) {
        return crflayer_pass(e, B, probs, image, params, log_out, result, s);
    });
}

// ---- one refinement, two consumers (train-s.prototxt:758-786: CRFLayer and DSRGLayer read the same blobs) ----
int dsrg_srg_last_crf_host(dsrg_engine *h, int B, const float *labels, const float *cues, double th1, double th2,
                           float *seeds_out) {
    return host_call(h, B, labels && cues && seeds_out, true, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_labels, labels, (size_t)B * e->M * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_cues, cues, n * sizeof(float), cudaMemcpyHostToDevice, s));
        // SRG on the raw marginals of the last pass, float64 clamp + renormalisation fused in (pylayers.py:328-344)
        if (int rc = srg_run(e, B, e->st_labels, e->Q0, e->st_cues, th1, th2, 1, e->st_out, nullptr, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(seeds_out, e->st_out, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    }, last_crf_held);
}

int dsrg_srg_last_crf_dev(dsrg_engine *h, const float *labels, const float *cues, int B, double th1, double th2,
                          float *seeds_out, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    return dev_call(h, B, s, labels && cues && seeds_out, [&](Engine *e) {
        if (int rc = last_crf_held(e, B)) return rc;
        // the device twin of the host entry point above: same kernels, queued behind the pass on the caller's stream
        return srg_run(e, B, labels, e->Q0, cues, th1, th2, 1, seeds_out, nullptr, s);
    });
}

int dsrg_crf_last_marginals_host(dsrg_engine *h, int B, float *out, int out_layout) {
    return host_call(h, B, out && layout_ok(out_layout), false, [&](Engine *e, cudaStream_t s) {
        if (int rc = meanfield_export(e, B, e->st_out, out_layout, s)) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(out, e->st_out, (size_t)B * e->M * e->N * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    }, last_crf_held);
}

int dsrg_crflayer_forward_host(dsrg_engine *h, int B, float *probs, const uint8_t *image,
                               const dsrg_crf_params *params, float *log_out, float *result) {
    return host_call(h, B, probs && image && params && log_out, true, [&](Engine *e, cudaStream_t s) {
        const size_t n = (size_t)B * e->M * e->N;
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, probs, n * sizeof(float), cudaMemcpyHostToDevice, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_image, image, (size_t)B * e->N * 3, cudaMemcpyHostToDevice, s));
        if (int rc = crflayer_pass(e, B, e->st_unary, e->st_image, params, e->st_out, result ? e->st_cues : nullptr, s))
            return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(log_out, e->st_out, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(probs, e->st_unary, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        if (result) DSRG_CUDA_TRY(cudaMemcpyAsync(result, e->st_cues, n * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}

int dsrg_engine_lattice_sizes(dsrg_engine *h, int B, int *v_spatial, int *v_bilateral) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_batch(e, B);
    if (rc) return rc;
    DSRG_CUDA_TRY(cudaDeviceSynchronize());
    if (v_spatial) DSRG_CUDA_TRY(cudaMemcpy(v_spatial, e->sp.vcount, sizeof(int), cudaMemcpyDeviceToHost));
    if (v_bilateral)
        DSRG_CUDA_TRY(cudaMemcpy(v_bilateral, e->bi.vcount, sizeof(int) * B, cudaMemcpyDeviceToHost));
    return DSRG_OK;
}

int dsrg_engine_lattice_tables(dsrg_engine *h, int which, int b, int *off_out, int *nbr_out) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_entry(e, 1, e && (which == 0 || which == 1) && b >= 0 && b < e->maxB);
    if (rc) return rc;
    const Lattice &L = which == 0 ? e->sp : e->bi;
    const int sb = L.shared ? 0 : b;
    DSRG_CUDA_TRY(cudaDeviceSynchronize());
    int V = 0, base = 0;
    DSRG_CUDA_TRY(cudaMemcpy(&V, L.vcount + sb, sizeof(int), cudaMemcpyDeviceToHost));
    if (!L.shared) DSRG_CUDA_TRY(cudaMemcpy(&base, L.rowbase + b, sizeof(int), cudaMemcpyDeviceToHost));
    const int dp1 = L.d + 1;
    if (off_out)
        DSRG_CUDA_TRY(cudaMemcpy(off_out, L.off + (size_t)sb * dp1 * L.N, sizeof(int32_t) * dp1 * L.N,
                                 cudaMemcpyDeviceToHost));
    if (nbr_out) {
        for (int j = 0; j < dp1; j++) {
            int *dst = nbr_out + (size_t)j * (V + 1) * 2;
            DSRG_CUDA_TRY(cudaMemcpy(dst, L.nbr + (size_t)j * L.nbr_stride + base, sizeof(int2) * (V + 1),
                                     cudaMemcpyDeviceToHost));
            for (int k = 0; k < 2 * (V + 1); k++) dst[k] -= base;
        }
    }
    return DSRG_OK;
}

int dsrg_engine_copy_norm(dsrg_engine *h, int which, int B, float *norm_out) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_entry(e, B, norm_out != nullptr);
    if (rc) return rc;
    DSRG_CUDA_TRY(cudaDeviceSynchronize());
    if (which == 0)
        DSRG_CUDA_TRY(cudaMemcpy(norm_out, e->sp.norm, sizeof(float) * e->N, cudaMemcpyDeviceToHost));
    else
        DSRG_CUDA_TRY(cudaMemcpy(norm_out, e->bi.norm, sizeof(float) * (size_t)B * e->N, cudaMemcpyDeviceToHost));
    return DSRG_OK;
}

int dsrg_engine_lattice_bary(dsrg_engine *h, int which, int b, float *bary_out) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_entry(e, 1, e && bary_out && (which == 0 || which == 1) && b >= 0 && b < e->maxB);
    if (rc) return rc;
    const Lattice &L = which == 0 ? e->sp : e->bi;
    const size_t n = (size_t)(L.d + 1) * L.N;
    DSRG_CUDA_TRY(cudaDeviceSynchronize());
    DSRG_CUDA_TRY(cudaMemcpy(bary_out, L.bary + (L.shared ? 0 : b) * n, sizeof(float) * n, cudaMemcpyDeviceToHost));
    return DSRG_OK;
}

int dsrg_engine_lattice_idle(dsrg_engine *h, int which, long long *counts_out) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_entry(e, 1, counts_out && (which == 0 || which == 1));
    if (rc) return rc;
    return lattice_idle(e, which == 0 ? e->sp : e->bi, counts_out);
}

int dsrg_engine_tile_views(dsrg_engine *h, int which, int b, int *nloc_out, uint8_t *hy_out, int *hdr_out,
                           uint16_t *loc_out, float *wn_out) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_entry(e, 1, e && wn_out && (which == 0 || which == 1) && b >= 0 && b < e->maxB);
    if (rc) return rc;
    if (e->MP > DSRG_MAX_LABELS && (nloc_out || hy_out || hdr_out || loc_out)) {
        set_error("the tile-local views are not built for %d labels (more than %d)", e->M, DSRG_MAX_LABELS);
        return DSRG_E_STATE;
    }
    const Lattice &L = which == 0 ? e->sp : e->bi;
    const size_t sb = L.shared ? 0 : b, n = (size_t)(L.d + 1) * L.N, nt = e->ntiles;
    DSRG_CUDA_TRY(cudaDeviceSynchronize());
    DSRG_CUDA_TRY(cudaMemcpy(wn_out, L.wn + sb * n, sizeof(float) * n, cudaMemcpyDeviceToHost));
    if (nloc_out) DSRG_CUDA_TRY(cudaMemcpy(nloc_out, L.tl_nloc + sb * nt, sizeof(int32_t) * nt, cudaMemcpyDeviceToHost));
    if (hy_out) DSRG_CUDA_TRY(cudaMemcpy(hy_out, L.tl_hy + sb * nt, nt, cudaMemcpyDeviceToHost));
    if (hdr_out)
        DSRG_CUDA_TRY(cudaMemcpy(hdr_out, L.tl_hdr + sb * nt * L.maxloc, sizeof(int2) * nt * L.maxloc,
                                 cudaMemcpyDeviceToHost));
    if (loc_out) DSRG_CUDA_TRY(cudaMemcpy(loc_out, L.tl_loc + sb * n, sizeof(uint16_t) * n, cudaMemcpyDeviceToHost));
    return DSRG_OK;
}

int dsrg_engine_tile_blocks(dsrg_engine *h, int which, int b, float *w_out, uint16_t *loc_out) {
    Engine *e = (Engine *)h;
    DeviceScope dev_scope(e);
    int rc = check_entry(e, 1, e && (which == 0 || which == 1) && b >= 0 && b < e->maxB);
    if (rc) return rc;
    if (e->MP > DSRG_MAX_LABELS) {
        set_error("the tile-local views are not built for %d labels (more than %d)", e->M, DSRG_MAX_LABELS);
        return DSRG_E_STATE;
    }
    const Lattice &L = which == 0 ? e->sp : e->bi;
    const size_t n = (size_t)e->ntiles * (L.d + 1) * kTileThreads, at = (L.shared ? 0 : b) * n;
    DSRG_CUDA_TRY(cudaDeviceSynchronize());
    if (w_out) DSRG_CUDA_TRY(cudaMemcpy(w_out, L.tl_w + at, sizeof(float) * n, cudaMemcpyDeviceToHost));
    if (loc_out) DSRG_CUDA_TRY(cudaMemcpy(loc_out, L.tl_li + at, sizeof(uint16_t) * n, cudaMemcpyDeviceToHost));
    return DSRG_OK;
}

// ------------------------------------------------------------------------------------------------
// DenseCRFWrapper-shaped object API (CRF/include/densecrf_wrapper.h:3-28)
// ------------------------------------------------------------------------------------------------
struct dsrg_densecrf {
    int W, H, M;
    std::vector<float> unary;          // negated energies == the `unary` of CRF()
    std::vector<unsigned char> image;
    dsrg_crf_params params;
    bool has_unary, has_pairwise;
};

// The reference builds one DenseCRFWrapper per image (CRF.py:21), so the objects must be cheap: they hold
// host copies of their inputs only, and borrow a process-wide batch-1 engine per label count -- sized for the
// largest image seen so far and re-shaped per call -- for the duration of inference()/map().
static std::mutex g_pool_mu;
static std::map<std::pair<int, int>, Engine *> g_pool;  // (device, label count) -> engine

static Engine *pool_engine(int H, int W, int M) {   // call with g_pool_mu held
    const int dev = dsrg_current_device();           // the caller's current device, like every drop-in
    Engine *&slot = g_pool[std::make_pair(dev, M)];
    Engine *e = slot;
    if (e && (H > e->Hcap || W > e->Wcap)) {
        H = H > e->Hcap ? H : e->Hcap;
        W = W > e->Wcap ? W : e->Wcap;
        dsrg_engine_destroy((dsrg_engine *)e);
        e = slot = nullptr;
    }
    if (!e) {
        const int Hc = (H + 63) / 64 * 64, Wc = (W + 63) / 64 * 64;   // head-room for slightly larger images
        e = slot = (Engine *)dsrg_engine_create(dev, 1, Hc, Wc, M);
        if (!e) return nullptr;
    }
    return e;
}

void dsrg_densecrf_release_engines(void) {
    std::lock_guard<std::mutex> lk(g_pool_mu);
    for (auto &kv : g_pool)
        if (kv.second) dsrg_engine_destroy((dsrg_engine *)kv.second);
    g_pool.clear();
}

dsrg_densecrf *dsrg_densecrf_create(int W, int H, int nlabels) {
    if (W < 1 || H < 1 || nlabels < 1 || nlabels > DSRG_MAX_LABELS_WIDE || (long long)H * W > (1ll << 24)) {
        set_error("bad shape (W=%d H=%d nlabels=%d; nlabels <= %d)", W, H, nlabels, DSRG_MAX_LABELS_WIDE);
        return nullptr;
    }
    if (dsrg_device_count() < 1) {
        set_error("no usable CUDA device: this library has no CPU fallback");
        return nullptr;
    }
    dsrg_densecrf *c = new (std::nothrow) dsrg_densecrf();
    if (!c) return nullptr;
    c->W = W;
    c->H = H;
    c->M = nlabels;
    c->has_unary = c->has_pairwise = false;
    return c;
}

void dsrg_densecrf_destroy(dsrg_densecrf *c) { delete c; }

int dsrg_densecrf_npixels(const dsrg_densecrf *c) { return c ? c->W * c->H : 0; }
int dsrg_densecrf_nlabels(const dsrg_densecrf *c) { return c ? c->M : 0; }

int dsrg_densecrf_set_unary_energy(dsrg_densecrf *c, const float *unary_costs) {
    if (!c || !unary_costs) {
        set_error("NULL pointer argument");
        return DSRG_E_INVALID;
    }
    const size_t n = (size_t)c->W * c->H * c->M;
    c->unary.resize(n);
    for (size_t i = 0; i < n; i++) c->unary[i] = -unary_costs[i];  // Q0 = softmax(-energy), densecrf.cpp:120
    c->has_unary = true;
    return DSRG_OK;
}

int dsrg_densecrf_add_pairwise_energy(dsrg_densecrf *c, float w1, float theta_alpha_1,
                                      float theta_alpha_2, float theta_betta_1, float theta_betta_2,
                                      float theta_betta_3, float w2, float theta_gamma_1,
                                      float theta_gamma_2, const unsigned char *im) {
    if (!c || !im) {
        set_error("NULL pointer argument");
        return DSRG_E_INVALID;
    }
    if (c->has_pairwise) {
        // DenseCRFWrapper::add_pairwise_energy APPENDS a Gaussian and a bilateral term on every call
        // (densecrf_wrapper.cpp:25-29); this object holds one pair, which is all CRF() ever adds (CRF.py:31-32)
        set_error("add_pairwise_energy was already called on this object: only one Gaussian + bilateral pair is supported");
        return DSRG_E_STATE;
    }
    c->params.w1 = w1;
    c->params.theta_alpha_x = theta_alpha_1;
    c->params.theta_alpha_y = theta_alpha_2;
    c->params.theta_beta_r = theta_betta_1;
    c->params.theta_beta_g = theta_betta_2;
    c->params.theta_beta_b = theta_betta_3;
    c->params.w2 = w2;
    c->params.theta_gamma_x = theta_gamma_1;
    c->params.theta_gamma_y = theta_gamma_2;
    c->image.assign(im, im + (size_t)c->W * c->H * 3);
    c->has_pairwise = true;
    return DSRG_OK;
}

// the engine an object borrows; the caller holds g_pool_mu until its export + copy are done
static int densecrf_engine(dsrg_densecrf *c, const void *out, Engine **e) {
    if (!c || !out) {
        set_error("bad argument (NULL pointer or value out of range)");
        return DSRG_E_INVALID;
    }
    *e = pool_engine(c->H, c->W, c->M);
    return *e ? DSRG_OK : DSRG_E_CUDA;
}

// runs the mean field on the borrowed engine, inside its host_call
static int densecrf_run(dsrg_densecrf *c, int n_iters, Engine *e, cudaStream_t s) {
    int rc = dsrg_engine_set_size((dsrg_engine *)e, c->H, c->W);
    if (rc) return rc;
    if (!c->has_unary) c->unary.assign((size_t)c->W * c->H * c->M, 0.0f);  // unary.fill(0), densecrf.cpp:117
    c->params.n_iters = n_iters;
    DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary, c->unary.data(), c->unary.size() * sizeof(float), cudaMemcpyHostToDevice, s));
    if (!c->has_pairwise) {
        // no pairwise term: every mean-field step reproduces Q = softmax(-unary) (densecrf.cpp:120-128 with an
        // empty pairwise list), which is what the reference returns
        dsrg_crf_params p0 = c->params;
        p0.n_iters = 0;
        return meanfield_run(e, 1, e->st_unary, DSRG_LAYOUT_NHWC, false, nullptr, p0, s);
    }
    DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_image, c->image.data(), c->image.size(), cudaMemcpyHostToDevice, s));
    return crf_pass(e, s, PassKind::densecrf, 1, &c->params, GraphKey(), [&]() {
        return crf_core(e, 1, e->st_unary, DSRG_LAYOUT_NHWC, false, nullptr, e->st_image, &c->params, s);
    });
}

int dsrg_densecrf_inference(dsrg_densecrf *c, int n_iters, float *probs_out) {
    std::lock_guard<std::mutex> lk(g_pool_mu);
    Engine *eng = nullptr;
    if (int rc = densecrf_engine(c, probs_out, &eng)) return rc;
    return host_call((dsrg_engine *)eng, 1, true, true, [&](Engine *e, cudaStream_t s) {
        int rc = densecrf_run(c, n_iters, e, s);
        if (rc || (rc = meanfield_export(e, 1, e->st_out, DSRG_LAYOUT_NHWC, s))) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(probs_out, e->st_out, c->unary.size() * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}

int dsrg_densecrf_map(dsrg_densecrf *c, int n_iters, int *labels) {
    std::lock_guard<std::mutex> lk(g_pool_mu);
    Engine *eng = nullptr;
    if (int rc = densecrf_engine(c, labels, &eng)) return rc;
    return host_call((dsrg_engine *)eng, 1, true, true, [&](Engine *e, cudaStream_t s) {
        int rc = densecrf_run(c, n_iters, e, s);
        if (rc || (rc = meanfield_export_map(e, 1, e->st_lmap, s))) return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(labels, e->st_lmap, (size_t)c->W * c->H * sizeof(int), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}

}  // extern "C"
