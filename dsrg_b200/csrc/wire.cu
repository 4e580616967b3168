// Host-buffer entry point of the full pass (dsrg_dsrg_forward_host) and its PCIe diet.
//
// The reference interface hands over host float32 blobs (Caffe Python layers): per batch of 64
// images at 321x321x21 that is 1.13 GB in and 1.11 GB out, which caps the end-to-end rate at the
// PCIe rate, far below the kernels.  Two of the four big planes are
// 0/1 masks stored as floats (the cues going in, pylayers.py:338-339, and the seeds coming out,
// :271-275) and the third (the in-place clamped probs, :312) differs from what the host already has
// only where a value was below 1e-4.  So the wire format is:
//   in : probs (float32, as is), cues as 1 bit/value (packed by host threads, SSE2 movemask)
//   out: seeds as 1 bit/value, clamp mask as 1 bit/value (the host applies probs[i] = 1e-4 itself)
// Everything is exact.  The seeds are the cues with grown pixels set to 1, so they are a 0/1 mask only when the cues
// are: a chunk whose cues are not all exactly 0 or 1 sends its cues and its seeds as floats (the clamp mask stays).
// The batch is cut into chunks that flow through three streams (H2D | kernels | D2H) while the
// calling thread packs the next chunk and unpacks finished ones.
#include <emmintrin.h>
#include <omp.h>
#include <unistd.h>

#include "common.cuh"

namespace dsrg {

// ---- device side -----------------------------------------------------------------------------
// one warp turns 32 consecutive values into one word (bit = lane), per image
__global__ void __launch_bounds__(kThreads)
k_bits_to_float(const uint32_t *bits, float *out, int n_img, int wpi) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_img) return;
    const uint32_t w = bits[(size_t)b * wpi + (i >> 5)];
    out[(size_t)b * n_img + i] = (w >> (i & 31)) & 1u ? 1.0f : 0.0f;
}

template <int MODE>  // 0: value != 0   1: value < kMinProb
__global__ void __launch_bounds__(kThreads)
k_float_to_bits(const float *in, uint32_t *bits, int n_img, int wpi) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const float v = i < n_img ? in[(size_t)b * n_img + i] : (MODE == 0 ? 0.0f : 1.0f);
    const unsigned m = __ballot_sync(0xffffffffu, MODE == 0 ? (v != 0.0f) : (v < kMinProb));
    if ((threadIdx.x & 31) == 0 && (i >> 5) < wpi) bits[(size_t)b * wpi + (i >> 5)] = m;
}

// ---- host side: ONE OpenMP region per chunk and operation (images x word blocks), SSE2 inside --
// (many small regions with many threads were measured to be slower than the PCIe time they save)
// CPUs this process may really use: the cgroup quota (the GPU boxes give a 128-thread host a 16-CPU
// quota; oversubscribing it was measured 2x slower), shared among the ranks of a torchrun launch.
static int cpu_budget() {
    // (not omp_get_max_threads(): torchrun exports OMP_NUM_THREADS=1; the num_threads clauses below override it)
    long onl = sysconf(_SC_NPROCESSORS_ONLN);
    int n = onl > 0 ? (int)onl : 1;
    if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        long long quota = 0, period = 0;
        char q[32] = {0};
        if (fscanf(f, "%31s %lld", q, &period) == 2 && q[0] != 'm' && period > 0) {
            quota = atoll(q);
            const int c = (int)((quota + period - 1) / period);
            if (c >= 1 && c < n) n = c;
        }
        fclose(f);
    }
    int ranks = 1;
    if (const char *ev = getenv("LOCAL_WORLD_SIZE")) ranks = atoi(ev) > 0 ? atoi(ev) : 1;
    n /= ranks;
    return n < 1 ? 1 : n;
}

static int host_threads() {
    static int n = 0;
    if (!n) {
        n = cpu_budget();
        if (n > 16) n = 16;
        if (const char *ev = getenv("DSRG_B200_HOST_THREADS")) n = atoi(ev);
        if (n < 1) n = 1;
    }
    return n;
}
// packing 0/1 planes on the host only pays when enough cores are available to outrun PCIe
static bool wire_worthwhile() { return host_threads() >= 6; }
constexpr int kWireBlocks = 16;  // word blocks per image

static inline void block_range(size_t total, int blk, size_t &lo, size_t &hi) {
    lo = total * blk / kWireBlocks;
    hi = total * (blk + 1) / kWireBlocks;
}

// words [w0, w1) of one plane; returns nonzero if a value is neither 0 nor 1
static int pack_words(const float *src, uint32_t *dst, size_t n, size_t w0, size_t w1) {
    int bad = 0;
    const size_t full = n / 32;
    const __m128 zero = _mm_setzero_ps(), one = _mm_set1_ps(1.0f);
    for (size_t w = w0; w < w1 && w < full; w++) {
        const float *p = src + w * 32;
        uint32_t m = 0;
        int ok = 0xF;
        for (int k = 0; k < 8; k++) {
            const __m128 v = _mm_loadu_ps(p + 4 * k);
            m |= (uint32_t)_mm_movemask_ps(_mm_cmpneq_ps(v, zero)) << (4 * k);
            ok &= _mm_movemask_ps(_mm_or_ps(_mm_cmpeq_ps(v, zero), _mm_cmpeq_ps(v, one)));
        }
        dst[w] = m;
        bad |= (ok != 0xF);
    }
    if (w1 > full && w0 <= full) {  // ragged last word
        uint32_t m = 0;
        for (size_t i = full * 32; i < n; i++) {
            const float v = src[i];
            if (v != 0.0f) m |= 1u << (i & 31);
            if (v != 0.0f && v != 1.0f) bad = 1;
        }
        dst[full] = m;
    }
    return bad;
}

// `nb` planes of n values each (plane stride n floats / wpi words); false if some value is not 0/1
static bool pack_mask(const float *src, uint32_t *dst, size_t n, size_t wpi, int nb = 1) {
    int bad = 0;
    const size_t words = (n + 31) / 32;
#pragma omp parallel for collapse(2) num_threads(host_threads()) schedule(static) reduction(| : bad)
    for (int b = 0; b < nb; b++)
        for (int blk = 0; blk < kWireBlocks; blk++) {
            size_t lo, hi;
            block_range(words, blk, lo, hi);
            bad |= pack_words(src + (size_t)b * n, dst + (size_t)b * wpi, n, lo, hi);
        }
    return !bad;
}

// Expand bits to 0.0f / 1.0f with non-temporal stores (a buffer we overwrite completely needs no
// read-for-ownership).  Planes start at arbitrary 4-byte offsets, so the first k floats are peeled and
// the bit stream is funnel-shifted by k: every 32-float group then starts on a 16-byte boundary.
static void unpack_block(const uint32_t *src, float *dst, size_t n, int blk) {
    const size_t words = (n + 31) / 32;
    size_t k = ((16 - (((uintptr_t)dst) & 15)) & 15) / 4;
    if (k > n) k = n;
    const size_t groups = (n - k) / 32;
    size_t j0, j1;
    block_range(groups, blk, j0, j1);
    if (blk == 0)
        for (size_t i = 0; i < k; i++) dst[i] = (src[0] >> i) & 1u ? 1.0f : 0.0f;
    float *base = dst + k;
    const __m128i sel = _mm_set_epi32(8, 4, 2, 1);
    const __m128 one = _mm_set1_ps(1.0f);
    for (size_t j = j0; j < j1; j++) {
        uint32_t m = src[j] >> k;
        if (k && j + 1 < words) m |= src[j + 1] << (32 - k);
        float *p = base + j * 32;
        for (int q = 0; q < 8; q++, m >>= 4) {
            const __m128i bitsv = _mm_and_si128(_mm_set1_epi32((int)(m & 0xF)), sel);
            _mm_stream_ps(p + 4 * q, _mm_and_ps(_mm_castsi128_ps(_mm_cmpeq_epi32(bitsv, sel)), one));
        }
    }
    _mm_sfence();
    if (blk == kWireBlocks - 1)
        for (size_t i = k + groups * 32; i < n; i++) dst[i] = (src[i >> 5] >> (i & 31)) & 1u ? 1.0f : 0.0f;
}

// probs[i] = 1e-4 wherever the device saw a value below the clamp (pylayers.py:312)
static void clamp_block(const uint32_t *src, float *probs, size_t n, int blk) {
    size_t w0, w1;
    block_range((n + 31) / 32, blk, w0, w1);
    for (size_t w = w0; w < w1; w++) {
        uint32_t m = src[w];
        while (m) {
            const int bit = __builtin_ctz(m);
            m &= m - 1;
            const size_t i = w * 32 + bit;
            if (i < n) probs[i] = kMinProb;
        }
    }
}

// seeds (bits -> floats) and the clamp mask of `nb` planes in one parallel region
static void unpack_planes(const uint32_t *sbits, float *seeds, const uint32_t *mbits, float *probs, size_t n,
                          size_t wpi, int nb) {
#pragma omp parallel for collapse(2) num_threads(host_threads()) schedule(static)
    for (int b = 0; b < nb; b++)
        for (int blk = 0; blk < kWireBlocks; blk++) {
            if (sbits) unpack_block(sbits + (size_t)b * wpi, seeds + (size_t)b * n, n, blk);
            if (mbits) clamp_block(mbits + (size_t)b * wpi, probs + (size_t)b * n, n, blk);
        }
}

static int ensure_wire(Engine *e) {
    if (e->d_cbits) return DSRG_OK;
    const size_t wpi = ((size_t)e->M * e->Ncap + 31) / 32, n = (size_t)e->maxB * wpi;
    int rc = 0;
    rc |= dalloc(e, &e->d_cbits, n);
    rc |= dalloc(e, &e->d_sbits, n);
    rc |= dalloc(e, &e->d_mbits, n);
    if (rc) return DSRG_E_NOMEM;
    DSRG_CUDA_TRY(numa_host_alloc((void **)&e->h_cbits, n * 4, e->device));
    DSRG_CUDA_TRY(numa_host_alloc((void **)&e->h_sbits, n * 4, e->device));
    DSRG_CUDA_TRY(numa_host_alloc((void **)&e->h_mbits, n * 4, e->device));
    return DSRG_OK;
}

void wire_free(Engine *e) {
    cudaFree(e->d_cbits);
    cudaFree(e->d_sbits);
    cudaFree(e->d_mbits);
    if (e->h_cbits) cudaFreeHost(e->h_cbits);
    if (e->h_sbits) cudaFreeHost(e->h_sbits);
    if (e->h_mbits) cudaFreeHost(e->h_mbits);
}

}  // namespace dsrg

using namespace dsrg;

// host-only utilities of the wire format, exported so that they can be unit-tested without a GPU
extern "C" int dsrg_wire_pack_mask(const float *src, uint32_t *dst, size_t n) {
    return pack_mask(src, dst, n, (n + 31) / 32, 1) ? 1 : 0;
}
extern "C" void dsrg_wire_unpack_mask(const uint32_t *src, float *dst, size_t n) {
    unpack_planes(src, dst, nullptr, nullptr, n, (n + 31) / 32, 1);
}
extern "C" void dsrg_wire_apply_clamp_mask(const uint32_t *src, float *probs, size_t n) {
    unpack_planes(nullptr, nullptr, src, probs, n, (n + 31) / 32, 1);
}

// srg_only: no CRF (probs are read-only, `renorm` as in dsrg_srg_batch_dev, optional label map out)
static int host_pass_impl(Engine *e, int B, const float *labels, float *probs, const float *cues,
                          const uint8_t *image, const dsrg_crf_params *params, double th1, double th2,
                          float *seeds_out, float *crf_out, bool srg_only, int renorm, int32_t *label_map_out);

static int host_pass(dsrg_engine *h, int B, const float *labels, float *probs, const float *cues,
                     const uint8_t *image, const dsrg_crf_params *params, double th1, double th2,
                     float *seeds_out, float *crf_out, bool srg_only, int renorm, int32_t *label_map_out) {
    const bool ok = labels && probs && cues && seeds_out && (srg_only || (image && params));
    return host_call(h, B, ok, true, [&](Engine *e, cudaStream_t) {
        const int rc = host_pass_impl(e, B, labels, probs, cues, image, params, th1, th2, seeds_out, crf_out, srg_only,
                                      renorm, label_map_out);
        if (rc != DSRG_OK) {
            // a chunk failed mid-pipeline: copies of earlier chunks may still be reading or writing the caller's
            // buffers -- wait for them before the error is reported (the outputs are then undefined, not in flight)
            cudaStreamSynchronize(e->in_stream);
            cudaStreamSynchronize(e->own_stream);
            cudaStreamSynchronize(e->out_stream);
            cudaGetLastError();
        }
        return rc;
    });
}

static int host_pass_impl(Engine *e, int B, const float *labels, float *probs, const float *cues,
                          const uint8_t *image, const dsrg_crf_params *params, double th1, double th2,
                          float *seeds_out, float *crf_out, bool srg_only, int renorm, int32_t *label_map_out) {
    int rc = ensure_wire(e);
    if (rc) return rc;
    // chunk schedule: a small first chunk gets the GPU going early, then full-size chunks
    const int chunk = e->host_chunk > 0 ? e->host_chunk : B;
    std::vector<int> cb0, cnb;
    if (const char *ev = getenv("DSRG_B200_HOST_SCHEDULE")) {  // e.g. "4,12,16,32": explicit chunk sizes (tuning aid)
        int b = 0;
        for (const char *p = ev; *p && b < B;) {
            int v = atoi(p);
            if (v < 1) break;
            if (v > e->maxB) v = e->maxB;
            if (v > B - b) v = B - b;
            cb0.push_back(b);
            cnb.push_back(v);
            b += v;
            while (*p && *p != ',') p++;
            if (*p == ',') p++;
        }
        while (b < B) {
            const int v = (B - b < chunk) ? B - b : chunk;
            cb0.push_back(b);
            cnb.push_back(v);
            b += v;
        }
    }
    if (cb0.empty()) {
        // default: five chunks that grow (5 | 9 | 13 | 17 | 20 of 64; boundaries at 8 %, 22 %, 42 %, 69 % of the batch).
        // The GPU is the slower stage of the pipeline at 321x321x21: a short first chunk gets it going early, later chunks must be big enough to keep
        // its kernels efficient, and the last one not so big that its D2H + unpack tail shows (tools/sweep_schedule.py
        // compares schedules).  A positive host_chunk caps the chunk size.
        const int cap = e->host_chunk > 0 ? e->host_chunk : B;
        const double edge[5] = {5.0 / 64, 14.0 / 64, 27.0 / 64, 44.0 / 64, 1.0};
        for (int b = 0, k = 0; b < B;) {
            int end = k < 5 ? (int)(edge[k] * B + 0.5) : B;
            k++;
            if (end <= b) continue;
            if (end > B || k >= 5) end = B;
            while (b < end) {
                int nb = end - b;
                if (nb > cap) nb = cap;
                cb0.push_back(b);
                cnb.push_back(nb);
                b += nb;
            }
        }
    }
    const int nchunks = (int)cb0.size();
    while ((int)e->pipe_events.size() < 3 * nchunks) {
        cudaEvent_t ev;
        DSRG_CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        e->pipe_events.push_back(ev);
    }
    cudaStream_t s_in = e->in_stream, s = e->own_stream, s_out = e->out_stream;
    const size_t img_elems = (size_t)e->M * e->N;
    const int n_img = (int)img_elems;
    const size_t wpi = (img_elems + 31) / 32;
    std::vector<char> packed(nchunks, 0);
    int next_unpack = 0;
    static const bool dbg = getenv("DSRG_B200_DEBUG_TIMING") != nullptr;
    // debug timeline (DSRG_B200_DEBUG_TIMING): per chunk H2D begin/end, kernels begin/end, D2H end
    std::vector<cudaEvent_t> tl;
    auto mark = [&](cudaStream_t st) {
        if (!dbg) return;
        cudaEvent_t ev;
        cudaEventCreate(&ev);
        cudaEventRecord(ev, st);
        tl.push_back(ev);
    };
    mark(s_in);  // time origin
    double t_pack = 0, t_unpack = 0, t_issue = 0, t_wait = 0, t0 = omp_get_wtime();
    // what travels as bits is decided per chunk: bit 0 cues (host packs), bit 1 seeds (host unpacks), bit 2 the
    // clamp mask of probs (host applies sparse writes -- cheap even with one or two threads, and it replaces a
    // full float D2H of the probs blob)
    enum { W_CUES = 1, W_SEEDS = 2, W_MASK = 4 };
    const bool many_threads = wire_worthwhile();
    auto finish_chunk = [&](int c) {  // host side of a finished chunk
        const int b0 = cb0[c], nb = cnb[c];
        if (!(packed[c] & (W_SEEDS | W_MASK))) return;
        const double tu = omp_get_wtime();
        unpack_planes((packed[c] & W_SEEDS) ? e->h_sbits + (size_t)b0 * wpi : nullptr, seeds_out + (size_t)b0 * img_elems,
                      (packed[c] & W_MASK) ? e->h_mbits + (size_t)b0 * wpi : nullptr, probs + (size_t)b0 * img_elems,
                      img_elems, wpi, nb);
        t_unpack += omp_get_wtime() - tu;
    };
    for (int c = 0; c < nchunks; c++) {
        const int b0 = cb0[c], nb = cnb[c];
        const size_t o = (size_t)b0 * img_elems, n = (size_t)nb * img_elems;
        // ---- H2D of what needs no packing starts first, the cues are packed meanwhile
        double ti = omp_get_wtime();
        mark(s_in);
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_labels + (size_t)b0 * e->M, labels + (size_t)b0 * e->M,
                                      (size_t)nb * e->M * sizeof(float), cudaMemcpyHostToDevice, s_in));
        DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_unary + o, probs + o, n * sizeof(float), cudaMemcpyHostToDevice, s_in));
        t_issue += omp_get_wtime() - ti;
        // ---- host: pack this chunk's cues (1 bit per value) unless they are not a 0/1 mask
        const double tp = omp_get_wtime();
        const bool ok = e->wire_compress != 0 && many_threads &&
                        pack_mask(cues + (size_t)b0 * img_elems, e->h_cbits + (size_t)b0 * wpi, img_elems, wpi, nb);
        // seeds keep every cue value as it is (pylayers.py:271-275): as bits only when the cues were 0/1
        const bool ok_s = ok;
        const bool ok_m = e->wire_compress != 0 && !srg_only;
        t_pack += omp_get_wtime() - tp;
        ti = omp_get_wtime();
        packed[c] = (char)((ok ? W_CUES : 0) | (ok_s ? W_SEEDS : 0) | (ok_m ? W_MASK : 0));
        if (ok)
            DSRG_CUDA_TRY(cudaMemcpyAsync(e->d_cbits + (size_t)b0 * wpi, e->h_cbits + (size_t)b0 * wpi,
                                          (size_t)nb * wpi * 4, cudaMemcpyHostToDevice, s_in));
        else
            DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_cues + o, cues + o, n * sizeof(float), cudaMemcpyHostToDevice, s_in));
        if (!srg_only)
            DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_image + (size_t)b0 * e->N * 3, image + (size_t)b0 * e->N * 3,
                                          (size_t)nb * e->N * 3, cudaMemcpyHostToDevice, s_in));
        DSRG_CUDA_TRY(cudaEventRecord(e->pipe_events[3 * c], s_in));
        mark(s_in);
        // ---- kernels
        DSRG_CUDA_TRY(cudaStreamWaitEvent(s, e->pipe_events[3 * c], 0));
        mark(s);
        dim3 gb(cdiv(n_img, kThreads), nb);
        // packed cues / seeds stay packed: the SRG kernels read and write the 1-bit planes directly (srg.cu)
        const uint32_t *cbits = ok ? e->d_cbits + (size_t)b0 * wpi : nullptr;
        uint32_t *sbits = ok_s ? e->d_sbits + (size_t)b0 * wpi : nullptr;
        if (ok_m)  // before the pass clamps the device copy in place
            DSRG_LAUNCH(e, T_WIRE, s,
                        k_float_to_bits<1><<<gb, kThreads, 0, s>>>(e->st_unary + o, e->d_mbits + (size_t)b0 * wpi, n_img, (int)wpi));
        if (srg_only)
            rc = srg_run(e, nb, e->st_labels + (size_t)b0 * e->M, e->st_unary + o, e->st_cues + o, th1, th2, renorm,
                         e->st_out + o, label_map_out ? e->st_lmap + (size_t)b0 * e->N : nullptr, s, cbits, sbits);
        else
            rc = dsrg_forward_core(e, nb, e->st_labels + (size_t)b0 * e->M, e->st_unary + o, e->st_cues + o, cbits,
                                   e->st_image + (size_t)b0 * e->N * 3, params, th1, th2, e->st_out + o, sbits, nullptr, s);
        if (rc) return rc;
        if (crf_out) {  // raw marginals of this chunk, parked in the (now consumed) cues staging area
            if ((rc = meanfield_export(e, nb, e->st_cues + o, DSRG_LAYOUT_NCHW, s))) return rc;
        }
        DSRG_CUDA_TRY(cudaEventRecord(e->pipe_events[3 * c + 1], s));
        mark(s);
        // ---- D2H
        DSRG_CUDA_TRY(cudaStreamWaitEvent(s_out, e->pipe_events[3 * c + 1], 0));
        if (ok_s)
            DSRG_CUDA_TRY(cudaMemcpyAsync(e->h_sbits + (size_t)b0 * wpi, e->d_sbits + (size_t)b0 * wpi,
                                          (size_t)nb * wpi * 4, cudaMemcpyDeviceToHost, s_out));
        else
            DSRG_CUDA_TRY(cudaMemcpyAsync(seeds_out + o, e->st_out + o, n * sizeof(float), cudaMemcpyDeviceToHost, s_out));
        // the reference mutates the probs blob in place (pylayers.py:312): hand the clamp back, as a mask or whole
        if (ok_m)
            DSRG_CUDA_TRY(cudaMemcpyAsync(e->h_mbits + (size_t)b0 * wpi, e->d_mbits + (size_t)b0 * wpi,
                                          (size_t)nb * wpi * 4, cudaMemcpyDeviceToHost, s_out));
        else if (!srg_only)
            DSRG_CUDA_TRY(cudaMemcpyAsync(probs + o, e->st_unary + o, n * sizeof(float), cudaMemcpyDeviceToHost, s_out));
        if (label_map_out)
            DSRG_CUDA_TRY(cudaMemcpyAsync(label_map_out + (size_t)b0 * e->N, e->st_lmap + (size_t)b0 * e->N,
                                          (size_t)nb * e->N * sizeof(int32_t), cudaMemcpyDeviceToHost, s_out));
        if (crf_out)
            DSRG_CUDA_TRY(cudaMemcpyAsync(crf_out + o, e->st_cues + o, n * sizeof(float), cudaMemcpyDeviceToHost, s_out));
        DSRG_CUDA_TRY(cudaEventRecord(e->pipe_events[3 * c + 2], s_out));
        mark(s_out);
        t_issue += omp_get_wtime() - ti;
        // ---- host: finish whatever has already come back while the GPU works on this chunk
        while (next_unpack < c && cudaEventQuery(e->pipe_events[3 * next_unpack + 2]) == cudaSuccess)
            finish_chunk(next_unpack++);
    }
    for (; next_unpack < nchunks; next_unpack++) {
        const double tw = omp_get_wtime();
        DSRG_CUDA_TRY(cudaEventSynchronize(e->pipe_events[3 * next_unpack + 2]));
        t_wait += omp_get_wtime() - tw;
        finish_chunk(next_unpack);
    }
    DSRG_CUDA_TRY(cudaStreamSynchronize(s_out));
    if (dbg && !tl.empty()) {
        fprintf(stderr, "[dsrg host pass] timeline (ms from the first H2D; chunk: h2d begin-end | kernels begin-end | d2h end):");
        for (int c = 0; c < nchunks; c++) {
            float t[5];
            for (int k = 0; k < 5; k++) cudaEventElapsedTime(&t[k], tl[0], tl[1 + 5 * c + k]);
            fprintf(stderr, "  [%d img: %.2f-%.2f | %.2f-%.2f | %.2f]", cnb[c], t[0], t[1], t[2], t[3], t[4]);
        }
        fprintf(stderr, "\n");
        for (auto ev : tl) cudaEventDestroy(ev);
    }
    if (dbg)
        fprintf(stderr, "[dsrg host pass] total %.2f ms: pack %.2f issue %.2f unpack %.2f wait %.2f (threads %d, chunks %d)\n",
                1e3 * (omp_get_wtime() - t0), 1e3 * t_pack, 1e3 * t_issue, 1e3 * t_unpack, 1e3 * t_wait, host_threads(),
                nchunks);
    return DSRG_OK;
}

extern "C" int dsrg_dsrg_forward_host(dsrg_engine *h, int B, const float *labels, float *probs,
                                      const float *cues, const uint8_t *image,
                                      const dsrg_crf_params *params, double th1, double th2,
                                      float *seeds_out, float *crf_out) {
    return host_pass(h, B, labels, probs, cues, image, params, th1, th2, seeds_out, crf_out, false, 1, nullptr);
}

extern "C" int dsrg_srg_batch_host(dsrg_engine *h, int B, const float *labels, const float *probs,
                                   const float *cues, double th1, double th2, int renorm, float *seeds_out,
                                   int32_t *label_map_out) {
    // probs are only read on this path (no clamp write-back), hence the const_cast
    return host_pass(h, B, labels, const_cast<float *>(probs), cues, nullptr, nullptr, th1, th2, seeds_out, nullptr,
                     true, renorm, label_map_out);
}
