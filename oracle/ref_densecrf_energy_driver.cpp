// oracle/ref_densecrf_energy_driver.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// extern "C" access to the REAL reference CRF's DenseCRF::klDivergence (densecrf.cpp:213-235) of given marginals, one
// term at a time: the CRF is built with nothing, with the unary alone, or with one pairwise term alone, so that the
// caller can separate the entropy, unary and pairwise terms by differences.  Compiled with the reference's own,
// unmodified CRF sources against oracle/eigen_shim into oracle/_ref/libdensecrf_energy_ref.so (oracle/energy.mk).
#include "densecrf.h"
#include "objective.h"

ObjectiveFunction::~ObjectiveFunction() {}

namespace {
MatrixXf matrix_of(const float *m, int M) {
    MatrixXf r(M, M);
    for (int i = 0; i < M; i++)
        for (int j = 0; j < M; j++) r(i, j) = m[i * M + j];
    return r;
}
LabelCompatibility *compat_of(float w, const float *mu, int M) {
    return mu ? (LabelCompatibility *)new MatrixCompatibility(matrix_of(mu, M)) : (LabelCompatibility *)new PottsCompatibility(w);
}
}  // namespace

extern "C" {
// klDivergence(q) of a DenseCRF2D(W, H, M), q [N][M] (pixel-major), with by `term`:
//   0  no term (the entropy alone)
//   1  setUnaryEnergy(unary_costs [N][M]) alone
//   2  addPairwiseGaussian(s[0], s[1], C) alone
//   3  addPairwiseBilateral(s[0], s[1], s[2], s[3], s[4], im [N][3], C) alone
//   4  addPairwiseEnergy(features [N][5], C) alone (DIAG_KERNEL, NORMALIZE_SYMMETRIC)
// where C is MatrixCompatibility(mu [M][M] row-major) or, with mu NULL, PottsCompatibility(w).
double ref_densecrf_kl(int W, int H, int M, const float *q, int term, const float *unary_costs, float w,
                       const float *mu, const float *s, const unsigned char *im, const float *features) {
    const int N = W * H;
    DenseCRF2D crf(W, H, M);
    if (term == 1) crf.setUnaryEnergy(Map<const MatrixXf>(unary_costs, M, N));
    if (term == 2) crf.addPairwiseGaussian(s[0], s[1], compat_of(w, mu, M));
    if (term == 3) crf.addPairwiseBilateral(s[0], s[1], s[2], s[3], s[4], im, compat_of(w, mu, M));
    if (term == 4) {
        MatrixXf f(5, N);
        for (int n = 0; n < N; n++)
            for (int j = 0; j < 5; j++) f(j, n) = features[n * 5 + j];
        crf.addPairwiseEnergy(f, compat_of(w, mu, M));
    }
    MatrixXf Q(M, N);
    for (int n = 0; n < N; n++)
        for (int l = 0; l < M; l++) Q(l, n) = q[n * M + l];
    return crf.klDivergence(Q);
}
}
