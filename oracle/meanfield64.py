"""oracle/meanfield64.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

DenseCRF::inference (densecrf.cpp:115-131; oracle/crf_oracle.c: oracle_crf_inference) restated in numpy on the
oracle's own lattices (``crf_oracle.DenseCRF(...).lattice(k)``: offset, bary, n1, n2), which are pinned bit for bit
to the reference's permutohedral.cpp and which the engine reproduces exactly (tests/test_gpu_lattice_order.py).  So
the device and this restatement run one algorithm on one lattice, and what is left between them is arithmetic.

In order, per iteration and per pairwise term (Gaussian, then bilateral, densecrf_wrapper.cpp:25-29):
``Q·norm``, splat, blur axes 0..d (row 0 is the missing neighbour), slice with ``alpha = 1/(1+2^-d)``, ``·norm``,
Potts ``-w``; then ``tmp = -unary - sum`` and exp-normalise.  ``norm`` is splat, blur and slice of ones, then
``1/sqrt(. + 1e-20)`` (pairwise.cpp:44-57).

Switches:

* ``dtype=np.float64``: the truth the device is measured against.
* ``dtype=np.float32, splat_order=None``: the oracle's own arithmetic -- sequential splat in incidence order, the
  blur in permutohedral.cpp's SSE form (``s = n1 + n2; hs = 0.5f*s; old + hs``) and for value sizes <= 2 (the norm
  pass, M <= 2) in the seq form with its double add (:505).  Its filter equals ``OracleLattice.compute`` bit for bit
  (tests/test_meanfield64_cpu.py).
* ``dtype=np.float32, splat_order=<seed>``: the same with each vertex's splat summed in a seeded shuffled order, a
  CPU model of the device's float atomics.
* ``arith="device"`` (float32): the device's own operation order (meanfield.cu, meanfield_wide.cu): folded weights
  ``wn = bary·norm`` and ``coef = w·alpha``, the splat ``wn·Q``, the slice as an fma chain onto the unary,
  ``exp`` with a seeded relative error of at most 2^-22 (``ex2.approx`` with its residual correction) and a
  reciprocal instead of a division.

``mutant`` injects one small error into the float32 restatement (see MUTANTS); the tests use it to show that their
bar sees errors of that size.
"""
import numpy as np
import scipy.sparse as sp

from . import crf_oracle

# name -> what the float32 restatement then does wrong
MUTANTS = {
    "axes_reversed": "blur axes taken d..0 instead of 0..d",
    "phantom_missing": "vertices only the phantom lanes touch treated as missing neighbours",
    "weight_rounded": "slice weight bary·alpha·norm rounded once more (norm folded into it)",
    "exp2_uncorrected": "exp(x) as exp2(x·log2e) without the residual correction",
    "values_fp16": "value rows rounded to fp16 after the splat",
}
EX2_REL = 2.0 ** -22      # relative error of ex2.approx with the residual correction (meanfield.cu: exp_neg)


class Lattice(object):
    """One pairwise term: the oracle's lattice of it, its Potts weight and alpha."""

    def __init__(self, lat, w):
        self.N, self.d, self.V = lat.N, lat.d, lat.M
        self.offset = lat.offset + 1                        # (N, d+1) value rows, row 0 = missing
        self.bary = lat.bary                                # (N, d+1) float32
        self.n1, self.n2 = lat.n1 + 1, lat.n2 + 1           # (d+1, V)
        self.w = float(w)
        self.rows = self.offset.ravel()
        self.cols = np.repeat(np.arange(self.N), self.d + 1)
        self._seq = np.argsort(self.rows, kind="stable")   # per vertex, its incidences in pixel order
        self.indptr = np.concatenate([[0], np.cumsum(np.bincount(self.rows, minlength=self.V + 1))])
        self._phantom_nbr = None

    def alpha(self, dtype):
        if dtype == np.float64:
            return 1.0 / (1.0 + 2.0 ** -self.d)
        return np.float32(1.0) / (np.float32(1.0) + np.float32(2.0 ** -self.d))   # permutohedral.cpp:510, :571

    def order(self, splat_order):
        if splat_order is None:
            return self._seq
        perm = np.random.RandomState(splat_order).permutation(self.rows.size)
        return perm[np.argsort(self.rows[perm], kind="stable")]

    def splat_matrix(self, weights, dtype, splat_order):
        """(V+1, N) CSR matrix whose product with X sums w·x per vertex in the chosen order (scipy's csr kernels
        add the entries of a row in storage order, in the result's dtype, from zero)."""
        o = self.order(splat_order)
        return sp.csr_matrix((weights.ravel()[o].astype(dtype), self.cols[o], self.indptr),
                             shape=(self.V + 1, self.N))

    def neighbours(self, mutant):
        if mutant != "phantom_missing":
            return self.n1, self.n2
        if self._phantom_nbr is None:
            real = np.zeros(self.V + 1, bool)
            real[self.rows] = True
            real[0] = True
            self._phantom_nbr = (np.where(real[self.n1], self.n1, 0), np.where(real[self.n2], self.n2, 0))
        return self._phantom_nbr

    def blur(self, v, seq, mutant=None):
        n1, n2 = self.neighbours(mutant)
        axes = range(self.d, -1, -1) if mutant == "axes_reversed" else range(self.d + 1)
        half = v.dtype.type(0.5)
        for j in axes:
            s = v[n1[j]] + v[n2[j]]
            new = np.empty_like(v)
            new[0] = 0
            if seq and v.dtype == np.float32:   # (float)((double)old + 0.5*(double)(n1 + n2)), :505
                new[1:] = (v[1:].astype(np.float64) + 0.5 * s.astype(np.float64)).astype(np.float32)
            else:
                new[1:] = v[1:] + half * s
            v = new
        return v

    def slice(self, v, seq, weights=None):
        """sum_r w_r · v[row_r]: SSE form (bary·alpha)·v, seq form (bary·v)·alpha; `weights` replaces bary·alpha."""
        alpha = self.alpha(v.dtype.type)
        acc = np.zeros((self.N, v.shape[1]), v.dtype)
        for r in range(self.d + 1):
            rows = v[self.offset[:, r]]
            if weights is not None:
                acc += weights[:, r, None] * rows
            elif seq:
                acc += (self.bary[:, r, None].astype(v.dtype) * rows) * alpha
            else:
                acc += (self.bary[:, r] * alpha).astype(v.dtype)[:, None] * rows
        return acc

    def filter(self, x, dtype, splat_order=None, mutant=None, slice_weights=None):
        """Permutohedral::compute (permutohedral.cpp:596-604) of x (N, vs): splat, blur, slice."""
        seq = x.shape[1] <= 2
        v = self.splat_matrix(self.bary, dtype, splat_order) @ x.astype(dtype)
        if mutant == "values_fp16":
            v = v.astype(np.float16).astype(dtype)
        return self.slice(self.blur(v, seq, mutant), seq, slice_weights)


class Problem(object):
    """The two lattices of one (H, W, 3) uint8 image under the pairwise parameters of a dsrg_crf_params, built once
    for every label count and every arithmetic."""

    def __init__(self, image, params):
        H, W = image.shape[:2]
        self.H, self.W, self.N = H, W, H * W
        c = crf_oracle.DenseCRF(W, H, 1)
        c.set_unary_energy(np.zeros(self.N, np.float32))
        c.add_pairwise_energy(params.w1, params.theta_alpha_x, params.theta_alpha_y, params.theta_beta_r,
                              params.theta_beta_g, params.theta_beta_b, params.w2, params.theta_gamma_x,
                              params.theta_gamma_y, np.ascontiguousarray(image).ravel())
        self.crf = c                       # keeps the oracle's lattices (and their compute()) alive
        self.lattices = [Lattice(c.lattice(0), params.w2), Lattice(c.lattice(1), params.w1)]
        self.n_iters = int(params.n_iters)
        self._norms = {}

    def norms(self, dtype, splat_order=None):
        """Per lattice, 1/sqrt(K·1 + 1e-20) (pairwise.cpp:44, :55-56); K·1 in the seq form (value size 1)."""
        key = (np.dtype(dtype).name, splat_order)
        if key not in self._norms:
            out = []
            for L in self.lattices:
                k1 = L.filter(np.ones((self.N, 1), dtype), dtype, splat_order)[:, 0]
                n = 1.0 / np.sqrt(k1.astype(np.float64) + 1e-20)
                out.append(n.astype(dtype))
            self._norms[key] = out
        return self._norms[key]

    def run(self, unary, n_iters=None, dtype=np.float64, splat_order=None, arith="oracle", mutant=None,
            exp_seed=0):
        """Q after 0, 1, ..., n_iters iterations (list of (H, W, M) arrays of `dtype`) for `unary` (H, W, M) float32
        log-probabilities -- what CRF() hands the CRF as -energy and what crf_dev takes."""
        n_iters = self.n_iters if n_iters is None else n_iters
        M = unary.shape[-1]
        U = np.ascontiguousarray(unary, np.float32).reshape(self.N, M).astype(dtype)   # -(-unary): exact
        norms = self.norms(dtype, splat_order)
        device = arith == "device"
        rng = np.random.RandomState(exp_seed)
        if device:
            assert dtype == np.float32 and mutant is None
            wn = [(L.bary * n[:, None]).astype(np.float32) for L, n in zip(self.lattices, norms)]
            S = [L.splat_matrix(w, dtype, splat_order) for L, w in zip(self.lattices, wn)]
            coef = [np.float32(np.float32(L.w) * L.alpha(np.float32)) for L in self.lattices]
        if mutant == "weight_rounded":
            sw = [((L.bary * L.alpha(np.float32)).astype(np.float32) * n[:, None]).astype(np.float32)
                  for L, n in zip(self.lattices, norms)]

        def softmax(t):
            mx = t.max(1, keepdims=True)
            x = t - mx
            if device:
                e = np.exp(x.astype(np.float64)) * (1.0 + rng.uniform(-EX2_REL, EX2_REL, x.shape))
                e = e.astype(np.float32)
            elif mutant == "exp2_uncorrected":
                e = np.exp2(x * np.float32(1.4426950408889634))
            else:                               # float32: expf rounded from float64, as glibc's expf nearly always
                e = np.exp(x.astype(np.float64)).astype(dtype)
            s = np.zeros(self.N, dtype)
            for k in range(M):                  # Eigen's sum -> a sequential sum (crf_oracle.c: exp_and_normalize)
                s += e[:, k]
            if device:
                return e * (np.float32(1.0) / s)[:, None]
            return e / s[:, None]

        Q = softmax(U)                          # densecrf.cpp:120
        out = [Q]
        for _ in range(n_iters):
            if device:
                t = U.copy()
                for L, Sk, c, w in zip(self.lattices, S, coef, wn):
                    v = L.blur(Sk @ Q, False)   # o + 0.5f*(a + d) at every label count
                    wr = (c * w).astype(np.float32)
                    for r in range(L.d + 1):   # t = fma(wr, v[row], t)
                        t = (wr[:, r, None].astype(np.float64) * v[L.offset[:, r]] + t).astype(np.float32)
            else:
                t = U.copy()                    # densecrf.cpp:123
                for k, (L, n) in enumerate(zip(self.lattices, norms)):
                    if mutant == "weight_rounded":
                        f = L.filter(Q * n[:, None], dtype, splat_order, slice_weights=sw[k])
                    else:
                        f = L.filter(Q * n[:, None], dtype, splat_order, mutant) * n[:, None]
                    t -= dtype(-L.w) * f        # Potts -w (labelcompatibility.cpp:46-48), densecrf.cpp:126
            Q = softmax(t)
            out.append(Q)
        return [q.reshape(self.H, self.W, M) for q in out]
