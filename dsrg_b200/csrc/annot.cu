// AnnotationLayer.forward on the device (SURVEY.md 8f rank 4): the step that feeds the path,
// pylayers/pylayers/pylayers.py:369-387:
//   top[0].data[...] = 0; top[1].data[...] = 0; top[2].data[...] = bottom[1].data        :371-373
//   top[0].data[i,0,0,0] = 1; top[0].data[i,0,0,labels_i] = 1                               :377-379
//   top[1].data[i, cues_i[0], cues_i[1], cues_i[2]] = 1                                      :381-382
//   if mirror: flip = choice(2)*2-1; top[1].data[i] = top[1].data[i,:,:,::flip]; same for top[2]   :384-387
// The pickle and the random draw stay on the host (the caller passes the index lists and the flip
// flags); the dense planes are produced in HBM, where dsrg_dsrg_forward_dev reads them.
#include <vector>

#include "common.cuh"

namespace dsrg {

__global__ void __launch_bounds__(kThreads)
k_annot_tags(const int32_t *tag_off, const int32_t *tags, float *labels, int M) {
    const int b = blockIdx.x;
    float *row = labels + (size_t)b * M;
    for (int l = threadIdx.x; l < M; l += blockDim.x) row[l] = l == 0 ? 1.0f : 0.0f;
    __syncthreads();
    for (int k = tag_off[b] + threadIdx.x; k < tag_off[b + 1]; k += blockDim.x) {
        int t = tags[k];
        if (t < 0) t += M;
        row[t] = 1.0f;
    }
}

// one thread per cue entry; `img` = image of the entry (entries are grouped by image)
__global__ void __launch_bounds__(kThreads)
k_annot_scatter(const int32_t *cue_off, const int32_t *idx, long long ktot, const int32_t *flip, float *cues,
                int B, int M, int H, int W) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= ktot) return;
    int lo = 0, hi = B;  // largest b with cue_off[b] <= k
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (cue_off[mid] <= k) lo = mid; else hi = mid;
    }
    int c = idx[k], y = idx[ktot + k], x = idx[2 * ktot + k];
    if (c < 0) c += M;
    if (y < 0) y += H;
    if (x < 0) x += W;
    if (flip && flip[lo]) x = W - 1 - x;
    cues[(((size_t)lo * M + c) * H + y) * W + x] = 1.0f;
}

__global__ void __launch_bounds__(kThreads)
k_annot_images(const float *in, float *out, const int32_t *flip, long long per_image, int Wi, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int b = (int)(i / per_image);
    const int x = (int)(i % Wi);
    const long long src = (flip && flip[b]) ? i - x + (Wi - 1 - x) : i;
    out[i] = in[src];
}

// host-side validation with numpy's rules: -dim <= index < dim, else IndexError
static int check_indices(const int32_t *v, long long n, int dim, const char *what) {
    for (long long k = 0; k < n; k++)
        if (v[k] < -dim || v[k] >= dim) {
            set_error("index %d is out of bounds for %s with size %d", v[k], what, dim);
            return DSRG_E_INVALID;
        }
    return DSRG_OK;
}

static int annotation_forward(Engine *e, int B, const int32_t *tag_off, const int32_t *tags,
                              const int32_t *cue_off, const int32_t *cue_idx, const int32_t *flip,
                              const float *images_in, int Hi, int Wi, float *labels_out, float *cues_out,
                              float *images_out, cudaStream_t s) {
    const long long nt = tag_off[B], nk = cue_off[B];
    if (tag_off[0] != 0 || cue_off[0] != 0 || nt < 0 || nk < 0 || (nt && !tags) || (nk && !cue_idx)) {
        set_error("bad offsets");
        return DSRG_E_INVALID;
    }
    for (int b = 0; b < B; b++)
        if (tag_off[b + 1] < tag_off[b] || cue_off[b + 1] < cue_off[b]) {
            set_error("offsets must be non-decreasing");
            return DSRG_E_INVALID;
        }
    int rc;
    if ((rc = check_indices(tags, nt, e->M, "the label axis"))) return rc;
    if ((rc = check_indices(cue_idx, nk, e->M, "axis 1 (class)"))) return rc;
    if ((rc = check_indices(cue_idx + nk, nk, e->H, "axis 2 (row)"))) return rc;
    if ((rc = check_indices(cue_idx + 2 * nk, nk, e->W, "axis 3 (column)"))) return rc;
    // device copy of the index lists: [tag_off B+1][cue_off B+1][flip B][tags nt][cue_idx 3*nk]
    const size_t n_ints = (size_t)(2 * (B + 1) + B) + nt + 3 * nk;
    if ((rc = grow_staging(e, (void **)&e->st_idx, &e->st_idx_cap, n_ints * sizeof(int32_t)))) return rc;
    std::vector<int32_t> pack(n_ints);
    int32_t *p = pack.data();
    memcpy(p, tag_off, sizeof(int32_t) * (B + 1));
    memcpy(p + (B + 1), cue_off, sizeof(int32_t) * (B + 1));
    for (int b = 0; b < B; b++) p[2 * (B + 1) + b] = flip ? (flip[b] != 0) : 0;
    if (nt) memcpy(p + 2 * (B + 1) + B, tags, sizeof(int32_t) * nt);
    if (nk) memcpy(p + 2 * (B + 1) + B + nt, cue_idx, sizeof(int32_t) * 3 * nk);
    // pageable source: the copy is staged before the call returns, `pack` may die afterwards
    DSRG_CUDA_TRY(cudaMemcpyAsync(e->st_idx, p, sizeof(int32_t) * n_ints, cudaMemcpyHostToDevice, s));
    const int32_t *d_tag_off = e->st_idx, *d_cue_off = e->st_idx + (B + 1), *d_flip = e->st_idx + 2 * (B + 1);
    const int32_t *d_tags = d_flip + B, *d_idx = d_tags + nt;
    DSRG_CUDA_TRY(cudaMemsetAsync(cues_out, 0, sizeof(float) * (size_t)B * e->M * e->N, s));
    DSRG_LAUNCH(e, T_ANNOT, s, k_annot_tags<<<B, 32, 0, s>>>(d_tag_off, d_tags, labels_out, e->M));
    if (nk)
        DSRG_LAUNCH(e, T_ANNOT, s,
                    k_annot_scatter<<<cdiv(nk, kThreads), kThreads, 0, s>>>(d_cue_off, d_idx, nk, flip ? d_flip : nullptr,
                                                                          cues_out, B, e->M, e->H, e->W));
    if (images_out) {
        const long long per = 3ll * Hi * Wi, n = per * B;
        DSRG_LAUNCH(e, T_ANNOT, s,
                    k_annot_images<<<cdiv(n, kThreads), kThreads, 0, s>>>(images_in, images_out, flip ? d_flip : nullptr,
                                                                        per, Wi, n));
    }
    DSRG_CUDA_TRY(cudaGetLastError());
    return DSRG_OK;
}

}  // namespace dsrg

using namespace dsrg;

// the pointers every call needs, and the image pair when the images are copied
static bool annot_args_ok(const int32_t *tag_off, const int32_t *cue_off, const float *images_in, int Hi, int Wi,
                          const float *labels_out, const float *cues_out, const float *images_out) {
    return tag_off && cue_off && labels_out && cues_out && (!images_out || (images_in && Hi >= 1 && Wi >= 1));
}

extern "C" int dsrg_annotation_forward_dev(dsrg_engine *h, int B, const int32_t *tag_offsets, const int32_t *tags,
                                           const int32_t *cue_offsets, const int32_t *cue_idx, const int32_t *flip,
                                           const float *images_in_dev, int Hi, int Wi, float *labels_out_dev,
                                           float *cues_out_dev, float *images_out_dev, void *stream) {
    const cudaStream_t s = (cudaStream_t)stream;
    // the mirror reads and writes whole rows: the two image buffers must be distinct
    const bool ok = annot_args_ok(tag_offsets, cue_offsets, images_in_dev, Hi, Wi, labels_out_dev, cues_out_dev,
                                  images_out_dev) && (!images_out_dev || images_in_dev != images_out_dev);
    return dev_call(h, B, s, ok, [&](Engine *e) {
        return annotation_forward(e, B, tag_offsets, tags, cue_offsets, cue_idx, flip, images_in_dev, Hi, Wi,
                                  labels_out_dev, cues_out_dev, images_out_dev, s);
    });
}

extern "C" int dsrg_annotation_forward_host(dsrg_engine *h, int B, const int32_t *tag_offsets, const int32_t *tags,
                                            const int32_t *cue_offsets, const int32_t *cue_idx, const int32_t *flip,
                                            const float *images_in, int Hi, int Wi, float *labels_out,
                                            float *cues_out, float *images_out) {
    const bool ok = annot_args_ok(tag_offsets, cue_offsets, images_in, Hi, Wi, labels_out, cues_out, images_out);
    return host_call(h, B, ok, false, [&](Engine *e, cudaStream_t s) {
        float *d_in = nullptr, *d_out = nullptr;
        const size_t nimg = images_out ? (size_t)B * 3 * Hi * Wi : 0;
        if (images_out) {
            if (int rc = grow_staging(e, (void **)&e->st_raw, &e->st_raw_cap, 2 * nimg * sizeof(float))) return rc;
            d_in = e->st_raw;
            d_out = e->st_raw + nimg;
            DSRG_CUDA_TRY(cudaMemcpyAsync(d_in, images_in, nimg * sizeof(float), cudaMemcpyHostToDevice, s));
        }
        if (int rc = annotation_forward(e, B, tag_offsets, tags, cue_offsets, cue_idx, flip, d_in, Hi, Wi,
                                        e->st_labels, e->st_cues, d_out, s))
            return rc;
        DSRG_CUDA_TRY(cudaMemcpyAsync(labels_out, e->st_labels, sizeof(float) * (size_t)B * e->M, cudaMemcpyDeviceToHost, s));
        DSRG_CUDA_TRY(cudaMemcpyAsync(cues_out, e->st_cues, sizeof(float) * (size_t)B * e->M * e->N, cudaMemcpyDeviceToHost, s));
        if (images_out)
            DSRG_CUDA_TRY(cudaMemcpyAsync(images_out, d_out, nimg * sizeof(float), cudaMemcpyDeviceToHost, s));
        return DSRG_OK;
    });
}
