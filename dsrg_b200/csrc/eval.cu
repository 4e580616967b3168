// Segmentation scoring on the device: the confusion matrix of the reference's evaluation tools.
//
//   ConfusionMatrix.generateM   training/tools/evaluate.py:61-68, training/tools/ap.py:65-72
//       for i in range(len(gt)): if gt[i] < nclass: m[gt[i], pred[i]] += 1.0
//   get_confusion_matrix        training/tools/test-coco.py:62-81 (np.bincount of gt * K + pred)
//
// An exact integer histogram of (gt, pred) pairs into a K x K matrix of uint64 counters, K <= DSRG_MAX_LABELS_WIDE.
// A pixel is binned iff gt < K and 0 <= pred < K.  gt >= K pixels are skipped; those other than 255 (the ignore
// label) are counted in invalid[0].  gt < K pixels whose pred is outside [0, K) are counted in invalid[1] (numpy
// would raise IndexError there).  Only integer atomics are used, so the result does not depend on the order.
//
// k_confusion streams gt (uint8) and pred (uint8 or int32) with 16-byte loads, 16 pixels per thread and step, in a
// persistent grid-stride loop.  Each CTA keeps the counters of one band of gt rows as u32 in shared memory; most
// pixels of a VOC image fall into bin (0,0), so a thread first run-length-encodes its 16 pixels and the warp then
// merges equal (bin, run) pairs with __match_any_sync, so one uniform region costs one shared atomic per warp.  At
// the end the non-zero counters are added to the global u64 matrix.  For K above ~110 the K x K counters do not
// fit in 48 KB: the gt rows are split into bands, one blockIdx.y per band, and every band re-reads the input.
#include <algorithm>
#include <new>

#include "common.cuh"

namespace dsrg {

constexpr int kEvalThreads = 256;
constexpr int kEvalSmemBytes = 48 * 1024;       // the histogram of one band of gt rows (no opt-in needed)
constexpr int kEvalVec = 16;                    // pixels per thread and step: one 16-byte load of gt
// Pixels one launch hands to each CTA at most, so no u32 shared counter can overflow before the flush.
constexpr size_t kEvalPixelsPerCta = size_t(1) << 30;

struct EvalArgs {
    const uint8_t *gt;
    const void *pred;
    size_t n;          // pixels
    int head;          // leading pixels before gt is 16-byte aligned (scalar prologue)
    long long nvec;    // 16-pixel vectors of the aligned body
    int K, rows;       // labels; gt rows per band
    unsigned long long *M;    // [K][K]
    unsigned long long *inv;  // [2]: gt >= K (not 255), pred outside [0, K)
};

// bin of one pixel within this CTA's band, or -1; counts the invalid pixels (each exactly once over the bands)
__device__ __forceinline__ int eval_bin(unsigned g, int p, int K, int r0, int rows, bool band0, unsigned &inv_gt,
                                        unsigned &inv_pred) {
    if (g >= (unsigned)K) {
        if (g != 255u && band0) inv_gt++;
        return -1;
    }
    const unsigned rel = g - (unsigned)r0;
    if (rel >= (unsigned)rows) return -1;
    if ((unsigned)p >= (unsigned)K) {
        inv_pred++;
        return -1;
    }
    return (int)rel * K + p;
}

template <typename T, bool VEC>
__device__ __forceinline__ void load_pred16(const T *p, int v[kEvalVec]) {
    if (VEC && sizeof(T) == 1) {
        const uint4 w = __ldcs(reinterpret_cast<const uint4 *>(p));
        const unsigned u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int j = 0; j < kEvalVec; j++) v[j] = (u[j >> 2] >> (8 * (j & 3))) & 0xFFu;
    } else if (VEC) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const int4 w = __ldcs(reinterpret_cast<const int4 *>(p) + q);
            v[4 * q] = w.x;
            v[4 * q + 1] = w.y;
            v[4 * q + 2] = w.z;
            v[4 * q + 3] = w.w;
        }
    } else {
#pragma unroll
        for (int j = 0; j < kEvalVec; j++) v[j] = (int)p[j];
    }
}

// VEC: pred is 16-byte aligned wherever gt is (else pred is read element by element)
template <typename T, bool VEC>
__global__ void __launch_bounds__(kEvalThreads)
k_confusion(EvalArgs a) {
    extern __shared__ unsigned hist[];
    const int r0 = blockIdx.y * a.rows, nbins = min(a.rows, a.K - r0) * a.K;
    const bool band0 = blockIdx.y == 0;
    for (int i = threadIdx.x; i < nbins; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const T *pred = static_cast<const T *>(a.pred);
    unsigned inv_gt = 0, inv_pred = 0;
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * blockDim.x;
    // every lane of a warp runs the same number of steps: the merge below is warp-synchronous
    for (long long v0 = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31); v0 < a.nvec; v0 += stride) {
        const long long v = v0 + lane;
        int cur = -1;
        unsigned run = 0;
        if (v < a.nvec) {
            const size_t px = (size_t)a.head + (size_t)v * kEvalVec;
            const uint4 gw = __ldcs(reinterpret_cast<const uint4 *>(a.gt + px));
            const unsigned gu[4] = {gw.x, gw.y, gw.z, gw.w};
            int pv[kEvalVec];
            load_pred16<T, VEC>(pred + px, pv);
#pragma unroll
            for (int j = 0; j < kEvalVec; j++) {
                const unsigned g = (gu[j >> 2] >> (8 * (j & 3))) & 0xFFu;
                const int b = eval_bin(g, pv[j], a.K, r0, a.rows, band0, inv_gt, inv_pred);
                if (b == cur) {
                    run++;
                } else {
                    if (cur >= 0) atomicAdd(&hist[cur], run);
                    cur = b;
                    run = 1;
                }
            }
        }
        // the last run of every lane: lanes with the same (bin, run) add once, run * their number
        const unsigned key = (cur < 0 ? 0xFFFFu : (unsigned)cur) | (run << 16);
        const unsigned peers = __match_any_sync(0xFFFFFFFFu, key);
        if (cur >= 0 && lane == __ffs(peers) - 1) atomicAdd(&hist[cur], run * __popc(peers));
    }
    // scalar prologue (pixels before gt is aligned) and epilogue (the last n mod 16), CTA 0 of each band
    if (blockIdx.x == 0) {
        const size_t tail0 = (size_t)a.head + (size_t)a.nvec * kEvalVec;
        for (size_t i = threadIdx.x; i < (size_t)a.head + (a.n - tail0); i += blockDim.x) {
            const size_t px = i < (size_t)a.head ? i : tail0 + (i - a.head);
            const int b = eval_bin(a.gt[px], (int)pred[px], a.K, r0, a.rows, band0, inv_gt, inv_pred);
            if (b >= 0) atomicAdd(&hist[b], 1u);
        }
    }
    const unsigned ig = __reduce_add_sync(0xFFFFFFFFu, inv_gt), ip = __reduce_add_sync(0xFFFFFFFFu, inv_pred);
    if (lane == 0) {
        if (ig) atomicAdd(&a.inv[0], (unsigned long long)ig);
        if (ip) atomicAdd(&a.inv[1], (unsigned long long)ip);
    }
    __syncthreads();
    unsigned long long *Mb = a.M + (size_t)r0 * a.K;   // the band's rows are contiguous in the matrix
    for (int i = threadIdx.x; i < nbins; i += blockDim.x) {
        const unsigned c = hist[i];
        if (c) atomicAdd(&Mb[i], (unsigned long long)c);
    }
}

// gt rows per band: all K when the K x K counters fit in shared memory
static int band_rows(int K) { return std::min(K, kEvalSmemBytes / (int)(sizeof(unsigned) * K)); }

struct Confusion {
    int device = 0, K = 0, sm_count = 132;
    unsigned long long *dM = nullptr;   // [K*K] matrix, then the 2 invalid counters
    // staging of the host variant: two pinned + device slots of kHostChunk pixels (gt, then pred as int32)
    static constexpr size_t kHostChunk = size_t(4) << 20;
    uint8_t *h_slot[2] = {nullptr, nullptr}, *d_slot[2] = {nullptr, nullptr};
    cudaStream_t copy_stream = nullptr, run_stream = nullptr;
    cudaEvent_t copied[2] = {nullptr, nullptr}, used[2] = {nullptr, nullptr};
    // order of the calls across streams: read / reset see every add before them
    cudaEvent_t order = nullptr;
    cudaStream_t last_stream = nullptr;
    bool last_valid = false;
};

// calls issued on different streams are ordered like an engine's passes (StreamScope), outside stream capture
struct ConfOrder {
    Confusion *c;
    cudaStream_t s;
    bool live = false;
    ConfOrder(Confusion *c_, cudaStream_t s_) : c(c_), s(s_) {
        cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(s, &st) != cudaSuccess) {
            cudaGetLastError();
            return;
        }
        if (st != cudaStreamCaptureStatusNone) return;
        live = true;
        if (c->last_valid && c->last_stream != s && cudaStreamWaitEvent(s, c->order, 0) != cudaSuccess) cudaGetLastError();
    }
    ~ConfOrder() {
        if (!live) return;
        if (cudaEventRecord(c->order, s) == cudaSuccess) {
            c->last_stream = s;
            c->last_valid = true;
        } else {
            cudaGetLastError();
        }
    }
};

static int confusion_launch(Confusion *c, size_t n, const uint8_t *gt, const void *pred, int pred_bytes,
                            cudaStream_t s) {
    const int rows = band_rows(c->K), bands = (c->K + rows - 1) / rows;
    const size_t smem = sizeof(unsigned) * rows * c->K;
    const bool vec = pred_bytes == 1 ? ((uintptr_t)gt & 15) == ((uintptr_t)pred & 15)
                                     : (((uintptr_t)pred + 4 * ((16 - ((uintptr_t)gt & 15)) & 15)) & 15) == 0;
    void (*kern)(EvalArgs) = pred_bytes == 1 ? (vec ? k_confusion<uint8_t, true> : k_confusion<uint8_t, false>)
                                             : (vec ? k_confusion<int32_t, true> : k_confusion<int32_t, false>);
    int occ = 0;
    DSRG_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kEvalThreads, smem));
    const int full = std::max(1, occ * c->sm_count / bands);
    const size_t chunk = (size_t)full * kEvalPixelsPerCta;
    for (size_t at = 0; at < n; at += chunk) {
        const size_t m = std::min(chunk, n - at);
        EvalArgs a;
        a.gt = gt + at;
        a.pred = (const char *)pred + at * pred_bytes;
        a.n = m;
        a.head = (int)std::min(m, (size_t)((16 - ((uintptr_t)a.gt & 15)) & 15));
        a.nvec = (long long)((m - a.head) / kEvalVec);
        a.K = c->K;
        a.rows = rows;
        a.M = c->dM;
        a.inv = c->dM + (size_t)c->K * c->K;
        const long long want = (a.nvec + kEvalThreads - 1) / kEvalThreads;
        const dim3 grid((unsigned)std::max(1LL, std::min<long long>(full, want)), bands);
        kern<<<grid, kEvalThreads, smem, s>>>(a);
        DSRG_CUDA_TRY(cudaGetLastError());
    }
    return DSRG_OK;
}

static void confusion_free(Confusion *c) {
    cudaFree(c->dM);
    for (int k = 0; k < 2; k++) {
        cudaFreeHost(c->h_slot[k]);
        cudaFree(c->d_slot[k]);
        if (c->copied[k]) cudaEventDestroy(c->copied[k]);
        if (c->used[k]) cudaEventDestroy(c->used[k]);
    }
    if (c->order) cudaEventDestroy(c->order);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    if (c->run_stream) cudaStreamDestroy(c->run_stream);
    delete c;
}

static int check_conf(const Confusion *c) {
    if (!c) {
        set_error("confusion object is NULL");
        return DSRG_E_INVALID;
    }
    return DSRG_OK;
}

static int check_add_args(size_t n, const uint8_t *gt, const void *pred, int pred_bytes) {
    if (pred_bytes != 1 && pred_bytes != 4) {
        set_error("pred_bytes must be 1 (uint8) or 4 (int32), not %d", pred_bytes);
        return DSRG_E_INVALID;
    }
    if (n > 0 && (!gt || !pred)) {
        set_error("NULL pointer argument");
        return DSRG_E_INVALID;
    }
    if (pred_bytes == 4 && ((uintptr_t)pred & 3)) {
        set_error("int32 pred must be 4-byte aligned");
        return DSRG_E_INVALID;
    }
    return DSRG_OK;
}

}  // namespace dsrg

using namespace dsrg;

extern "C" dsrg_confusion *dsrg_confusion_create(int device, int K) {
    if (K < 1 || K > DSRG_MAX_LABELS_WIDE) {
        set_error("bad label count %d (1 <= K <= %d)", K, DSRG_MAX_LABELS_WIDE);
        return nullptr;
    }
    int ndev = 0;
    if (device < 0) device = dsrg_current_device();
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) {
        cudaGetLastError();
        set_error("no usable CUDA device %d (visible devices: %d): this library has no CPU fallback", device, ndev);
        return nullptr;
    }
    Confusion *c = new (std::nothrow) Confusion();
    if (!c) return nullptr;
    c->device = device;
    c->K = K;
    DeviceScope dev_scope(c->device);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) {
        cudaGetLastError();
        set_error("device %d is not sm_90; this build contains sm_90a code only", device);
        delete c;
        return nullptr;
    }
    c->sm_count = prop.multiProcessorCount;
    const size_t mbytes = sizeof(unsigned long long) * ((size_t)K * K + 2);
    bool ok = cudaMalloc(&c->dM, mbytes) == cudaSuccess && cudaMemset(c->dM, 0, mbytes) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&c->order, cudaEventDisableTiming) == cudaSuccess;
    if (!ok) {
        cudaGetLastError();
        set_error("allocating the %dx%d confusion matrix failed", K, K);
        confusion_free(c);
        return nullptr;
    }
    return (dsrg_confusion *)c;
}

extern "C" void dsrg_confusion_destroy(dsrg_confusion *h) {
    Confusion *c = (Confusion *)h;
    if (!c) return;
    DeviceScope dev_scope(c->device);
    cudaDeviceSynchronize();
    confusion_free(c);
}

extern "C" int dsrg_confusion_reset(dsrg_confusion *h, void *stream) {
    Confusion *c = (Confusion *)h;
    int rc = check_conf(c);
    if (rc) return rc;
    DeviceScope dev_scope(c->device);
    cudaStream_t s = (cudaStream_t)stream;
    ConfOrder order(c, s);
    DSRG_CUDA_TRY(cudaMemsetAsync(c->dM, 0, sizeof(unsigned long long) * ((size_t)c->K * c->K + 2), s));
    return DSRG_OK;
}

extern "C" int dsrg_confusion_add_dev(dsrg_confusion *h, size_t n, const uint8_t *gt_dev, const void *pred_dev,
                                      int pred_bytes, void *stream) {
    Confusion *c = (Confusion *)h;
    int rc = check_conf(c);
    if (rc || (rc = check_add_args(n, gt_dev, pred_dev, pred_bytes))) return rc;
    if (n == 0) return DSRG_OK;
    DeviceScope dev_scope(c->device);
    cudaStream_t s = (cudaStream_t)stream;
    ConfOrder order(c, s);
    return confusion_launch(c, n, gt_dev, pred_dev, pred_bytes, s);
}

// Chunks of kHostChunk pixels go through two pinned / device slot pairs: the host copies chunk k+1 into its pinned
// slot and the copy stream moves it over PCIe while the run stream counts chunk k.
extern "C" int dsrg_confusion_add_host(dsrg_confusion *h, size_t n, const uint8_t *gt, const void *pred,
                                       int pred_bytes) {
    Confusion *c = (Confusion *)h;
    int rc = check_conf(c);
    if (rc || (rc = check_add_args(n, gt, pred, pred_bytes))) return rc;
    if (n == 0) return DSRG_OK;
    DeviceScope dev_scope(c->device);
    const size_t slot_bytes = Confusion::kHostChunk * 5;   // gt bytes, then up to 4 pred bytes per pixel
    if (!c->h_slot[0]) {
        bool ok = cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking) == cudaSuccess &&
                  cudaStreamCreateWithFlags(&c->run_stream, cudaStreamNonBlocking) == cudaSuccess;
        for (int k = 0; k < 2 && ok; k++)
            ok = cudaHostAlloc((void **)&c->h_slot[k], slot_bytes, cudaHostAllocDefault) == cudaSuccess &&
                 cudaMalloc((void **)&c->d_slot[k], slot_bytes) == cudaSuccess &&
                 cudaEventCreateWithFlags(&c->copied[k], cudaEventDisableTiming) == cudaSuccess &&
                 cudaEventCreateWithFlags(&c->used[k], cudaEventDisableTiming) == cudaSuccess &&
                 cudaEventRecord(c->copied[k], c->copy_stream) == cudaSuccess &&
                 cudaEventRecord(c->used[k], c->run_stream) == cudaSuccess;
        if (!ok) {
            cudaGetLastError();
            set_error("allocating the host staging of the confusion matrix failed");
            return DSRG_E_NOMEM;
        }
    }
    cudaStream_t s = c->run_stream;
    {
        ConfOrder order(c, s);
        const uint8_t *p8 = static_cast<const uint8_t *>(pred);
        int k = 0;
        for (size_t at = 0; at < n; at += Confusion::kHostChunk, k ^= 1) {
            const size_t m = std::min(Confusion::kHostChunk, n - at);
            uint8_t *hs = c->h_slot[k], *ds = c->d_slot[k];
            const size_t pred_off = Confusion::kHostChunk;   // 16-byte aligned, so is the device pred
            DSRG_CUDA_TRY(cudaEventSynchronize(c->copied[k]));   // the slot's previous H2D has read it
            memcpy(hs, gt + at, m);
            memcpy(hs + pred_off, p8 + at * pred_bytes, m * pred_bytes);
            DSRG_CUDA_TRY(cudaStreamWaitEvent(c->copy_stream, c->used[k], 0));   // the kernel of chunk k-2 is done
            DSRG_CUDA_TRY(cudaMemcpyAsync(ds, hs, m, cudaMemcpyHostToDevice, c->copy_stream));
            DSRG_CUDA_TRY(cudaMemcpyAsync(ds + pred_off, hs + pred_off, m * pred_bytes, cudaMemcpyHostToDevice,
                                          c->copy_stream));
            DSRG_CUDA_TRY(cudaEventRecord(c->copied[k], c->copy_stream));
            DSRG_CUDA_TRY(cudaStreamWaitEvent(s, c->copied[k], 0));
            if ((rc = confusion_launch(c, m, ds, ds + pred_off, pred_bytes, s))) return rc;
            DSRG_CUDA_TRY(cudaEventRecord(c->used[k], s));
        }
    }
    // the caller's arrays are only borrowed for the call: the last copies out of the pinned slots are done, but
    // wait for the counting too, so that errors surface here
    DSRG_CUDA_TRY(cudaStreamSynchronize(s));
    return DSRG_OK;
}

extern "C" int dsrg_confusion_read(dsrg_confusion *h, uint64_t *matrix_out, uint64_t *invalid_out) {
    Confusion *c = (Confusion *)h;
    int rc = check_conf(c);
    if (rc) return rc;
    if (!matrix_out && !invalid_out) {
        set_error("NULL pointer argument");
        return DSRG_E_INVALID;
    }
    DeviceScope dev_scope(c->device);
    if (c->last_valid) DSRG_CUDA_TRY(cudaEventSynchronize(c->order));
    const size_t kk = (size_t)c->K * c->K;
    if (matrix_out) DSRG_CUDA_TRY(cudaMemcpy(matrix_out, c->dM, kk * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    if (invalid_out) DSRG_CUDA_TRY(cudaMemcpy(invalid_out, c->dM + kk, 2 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    return DSRG_OK;
}
