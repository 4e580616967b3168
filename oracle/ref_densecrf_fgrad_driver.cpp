// oracle/ref_densecrf_fgrad_driver.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// extern "C" access to the REAL reference CRF's gradient to caller-given bilateral features: a DenseCRF with the
// Gaussian term of DenseCRFWrapper and a second term added as addPairwiseEnergy(features, PottsCompatibility or
// MatrixCompatibility, FULL_KERNEL) at P = I, whose kernel_grad is featureGradient fg times f^T (pairwise.cpp).
// Compiled with the reference's own, unmodified CRF sources against oracle/eigen_shim into
// oracle/_ref/libdensecrf_fgrad_ref.so (oracle/fgrad.mk).
#include "densecrf.h"
#include "objective.h"
#include "unary.h"

ObjectiveFunction::~ObjectiveFunction() {}

namespace {
// as in ref_densecrf_kgrad_driver.cpp
class GivenUnary : public UnaryEnergy {
    MatrixXf u_;

public:
    explicit GivenUnary(const MatrixXf &u) : u_(u) {}
    MatrixXf get() const { return u_; }
    VectorXf gradient(const MatrixXf &b) const {
        VectorXf r(b.rows() * b.cols());
        for (int i = 0; i < b.rows() * b.cols(); i++) r[i] = b.data()[i];
        return r;
    }
};
class GivenGradient : public ObjectiveFunction {
    MatrixXf g_;

public:
    explicit GivenGradient(const MatrixXf &g) : g_(g) {}
    double evaluate(MatrixXf &d_mul_Q, const MatrixXf &Q) const {
        d_mul_Q.resize(Q.rows(), Q.cols());
        double r = 0;
        for (int i = 0; i < Q.rows() * Q.cols(); i++) {
            d_mul_Q.data()[i] = g_.data()[i] * Q.data()[i];
            r += d_mul_Q.data()[i];
        }
        return r;
    }
};
MatrixXf matrix_of(const float *m, int M) {
    MatrixXf r(M, M);
    for (int i = 0; i < M; i++)
        for (int j = 0; j < M; j++) r(i, j) = m[i * M + j];
    return r;
}
}  // namespace

extern "C" {
// unary_costs, grad_q [N][M]; features [N][5] (pixel-major, the bilateral term's features as they are); mu_bi / mu_sp
// [M][M] row-major or NULL for PottsCompatibility(w1) / (w2).
//   kernel_grad_out[27] = kernel_grad: the Gaussian term's DIAG dL/dp (x, y), then the feature term's FULL dL/dP,
//                         fg f^T (5 x 5) in Eigen's column-major order
void ref_densecrf_fgrad(int W, int H, int M, const float *unary_costs, float w1, const float *mu_bi,
                        const float *features, float w2, const float *mu_sp, float tg1, float tg2, int n_iters,
                        const float *grad_q, float *kernel_grad_out) {
    const int N = W * H;
    DenseCRF2D crf(W, H, M);
    crf.setUnaryEnergy(new GivenUnary(Map<const MatrixXf>(unary_costs, M, N)));
    crf.addPairwiseGaussian(tg1, tg2, mu_sp ? (LabelCompatibility *)new MatrixCompatibility(matrix_of(mu_sp, M))
                                            : (LabelCompatibility *)new PottsCompatibility(w2));
    MatrixXf f(5, N);
    for (int n = 0; n < N; n++)
        for (int j = 0; j < 5; j++) f(j, n) = features[n * 5 + j];
    crf.addPairwiseEnergy(f, mu_bi ? (LabelCompatibility *)new MatrixCompatibility(matrix_of(mu_bi, M))
                                   : (LabelCompatibility *)new PottsCompatibility(w1),
                          FULL_KERNEL);
    GivenGradient obj(Map<const MatrixXf>(grad_q, M, N));
    VectorXf kg;
    crf.gradient(n_iters, obj, nullptr, nullptr, &kg);
    for (int i = 0; i < 27 && i < kg.rows(); i++) kernel_grad_out[i] = kg[i];
}
}
