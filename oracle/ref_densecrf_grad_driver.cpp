// oracle/ref_densecrf_grad_driver.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// extern "C" access to the REAL reference CRF's DenseCRF::gradient (densecrf.cpp:238-297), which DenseCRFWrapper
// leaves unused: compiled with the reference's own, unmodified CRF sources (the list oracle/Makefile compiles into
// libdensecrf_ref.so) against the Eigen stand-in in oracle/eigen_shim into oracle/_ref/libdensecrf_grad_ref.so
// (oracle/grad.mk).
#include "densecrf.h"
#include "objective.h"
#include "unary.h"

// objective.cpp is not part of the build (it needs more of Eigen than the stand-in has); the gradient only needs the
// abstract base's destructor
ObjectiveFunction::~ObjectiveFunction() {}

namespace {
// a constant unary whose parameter gradient is b itself, i.e. dL/d(energy) in [N][M] order
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
// L = sum G Q for a given G = dL/dQ_T: d_mul_Q = G * Q
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
}  // namespace

extern "C" {
// DenseCRF::gradient of the CRF DenseCRFWrapper builds (Gaussian term first, densecrf_wrapper.cpp:25-29) for the
// energies `unary_costs` [N][M] and an upstream G = dL/dQ_T [N][M]: unary_grad_out [N][M] = dL/d(energy),
// lbl_grad_out[2] = {dL/dw2, dL/dw1}.  kernel_grad is not asked for.
void ref_densecrf_gradient(int W, int H, int M, const float *unary_costs, float w1, float ta1, float ta2, float tb1,
                           float tb2, float tb3, float w2, float tg1, float tg2, const unsigned char *im, int n_iters,
                           const float *grad_q, float *unary_grad_out, float *lbl_grad_out) {
    DenseCRF2D crf(W, H, M);
    crf.setUnaryEnergy(new GivenUnary(Map<const MatrixXf>(unary_costs, M, W * H)));
    crf.addPairwiseGaussian(tg1, tg2, new PottsCompatibility(w2));
    crf.addPairwiseBilateral(ta1, ta2, tb1, tb2, tb3, im, new PottsCompatibility(w1));
    GivenGradient obj(Map<const MatrixXf>(grad_q, M, W * H));
    VectorXf ug, lg;
    crf.gradient(n_iters, obj, &ug, &lg, nullptr);
    for (int i = 0; i < M * W * H; i++) unary_grad_out[i] = ug[i];
    lbl_grad_out[0] = lg[0];
    lbl_grad_out[1] = lg[1];
}
}
