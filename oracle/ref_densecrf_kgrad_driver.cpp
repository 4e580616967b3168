// oracle/ref_densecrf_kgrad_driver.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// extern "C" access to the REAL reference CRF's kernel_grad: DenseCRF::gradient (densecrf.cpp:238-297) asked for its
// third output, under the reference's default DIAG_KERNEL and NORMALIZE_SYMMETRIC, with Potts or MatrixCompatibility
// terms.  Compiled with the reference's own, unmodified CRF sources against oracle/eigen_shim into
// oracle/_ref/libdensecrf_kgrad_ref.so (oracle/kgrad.mk).
#include "densecrf.h"
#include "objective.h"
#include "unary.h"

ObjectiveFunction::~ObjectiveFunction() {}

namespace {
// as in ref_densecrf_grad_driver.cpp: a constant unary whose parameter gradient is b itself ([N][M])
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
// L = sum G Q for a given G = dL/dQ_T
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
// [M][M] row-major -> MatrixXf
MatrixXf matrix_of(const float *m, int M) {
    MatrixXf r(M, M);
    for (int i = 0; i < M; i++)
        for (int j = 0; j < M; j++) r(i, j) = m[i * M + j];
    return r;
}
}  // namespace

extern "C" {
// The CRF of DenseCRFWrapper (Gaussian term first, densecrf_wrapper.cpp:25-29) for the energies `unary_costs` [N][M]
// and an upstream G = dL/dQ_T [N][M].  mu_bi / mu_sp ([M][M] row-major, the reference's MatrixCompatibility, which
// applies (m + m^T) / 2) or, when NULL, PottsCompatibility(w1) / PottsCompatibility(w2).
//   kernel_grad_out[7] = kernel_grad: dL/dp of the DIAG parameters in the order the kernels are added (spatial x, y,
//                        then bilateral x, y, r, g, b)
void ref_densecrf_kgrad(int W, int H, int M, const float *unary_costs, float w1, const float *mu_bi, float ta1,
                        float ta2, float tb1, float tb2, float tb3, float w2, const float *mu_sp, float tg1, float tg2,
                        const unsigned char *im, int n_iters, const float *grad_q, float *kernel_grad_out) {
    DenseCRF2D crf(W, H, M);
    crf.setUnaryEnergy(new GivenUnary(Map<const MatrixXf>(unary_costs, M, W * H)));
    crf.addPairwiseGaussian(tg1, tg2, mu_sp ? (LabelCompatibility *)new MatrixCompatibility(matrix_of(mu_sp, M))
                                            : (LabelCompatibility *)new PottsCompatibility(w2));
    crf.addPairwiseBilateral(ta1, ta2, tb1, tb2, tb3, im,
                             mu_bi ? (LabelCompatibility *)new MatrixCompatibility(matrix_of(mu_bi, M))
                                   : (LabelCompatibility *)new PottsCompatibility(w1));
    GivenGradient obj(Map<const MatrixXf>(grad_q, M, W * H));
    VectorXf kg;
    crf.gradient(n_iters, obj, nullptr, nullptr, &kg);
    for (int i = 0; i < 7 && i < kg.rows(); i++) kernel_grad_out[i] = kg[i];
}
}
