// oracle/ref_densecrf_compat_driver.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// extern "C" access to the REAL reference CRF with a MatrixCompatibility on both pairwise terms
// (labelcompatibility.cpp:64-108): DenseCRF::inference (densecrf.cpp:115-131) and DenseCRF::gradient
// (densecrf.cpp:238-297) with its packed lbl_cmp_grad.  Compiled with the reference's own, unmodified CRF sources
// against oracle/eigen_shim into oracle/_ref/libdensecrf_compat_ref.so (oracle/compat.mk).
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
// The CRF of DenseCRFWrapper (Gaussian term first, densecrf_wrapper.cpp:25-29) with MatrixCompatibility(mu_sp) and
// MatrixCompatibility(mu_bi) in place of the Potts terms, for the energies `unary_costs` [N][M]:
//   q_out [N][M]          = inference(n_iters)
//   unary_grad_out [N][M] = dL/d(energy) for L = sum grad_q Q_T
//   lbl_grad_out          = lbl_cmp_grad, M (M + 1) / 2 entries per term (upper triangle, row-major, g(i,j) + g(j,i)
//                           off the diagonal), the Gaussian term's first
void ref_densecrf_compat(int W, int H, int M, const float *unary_costs, const float *mu_bi, float ta1, float ta2,
                         float tb1, float tb2, float tb3, const float *mu_sp, float tg1, float tg2,
                         const unsigned char *im, int n_iters, const float *grad_q, float *q_out,
                         float *unary_grad_out, float *lbl_grad_out) {
    DenseCRF2D crf(W, H, M);
    crf.setUnaryEnergy(new GivenUnary(Map<const MatrixXf>(unary_costs, M, W * H)));
    crf.addPairwiseGaussian(tg1, tg2, new MatrixCompatibility(matrix_of(mu_sp, M)));
    crf.addPairwiseBilateral(ta1, ta2, tb1, tb2, tb3, im, new MatrixCompatibility(matrix_of(mu_bi, M)));
    MatrixXf Q = crf.inference(n_iters);
    for (int i = 0; i < M * W * H; i++) q_out[i] = Q.data()[i];
    GivenGradient obj(Map<const MatrixXf>(grad_q, M, W * H));
    VectorXf ug, lg;
    crf.gradient(n_iters, obj, &ug, &lg, nullptr);
    for (int i = 0; i < M * W * H; i++) unary_grad_out[i] = ug[i];
    for (int i = 0; i < lg.rows(); i++) lbl_grad_out[i] = lg[i];
}
}
