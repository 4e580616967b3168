"""oracle/sec_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

numpy restatements of SEC's seeding and expansion losses, SeedLossLayer (pylayers/pylayers/pylayers.py:95-118)
and ExpandLossLayer (:183-233), forward and analytic gradient, for any number of classes M (channel 0 =
background), plane size H x W and GWRP decay q.  The reference builds both with Theano 0.8.2; its class bodies are
executed in place by oracle/sec_layers.py, and tests/golden/sec_layers_ref.npz freezes those outputs at the
reference's shape (N, 21, 41, 41), which pins these restatements at 1e-12 in float64.

The gradients are what Theano's T.grad builds (restated from Theano's source, not from a Theano run): the
gradient of a sorted position goes to the element argsort put there, the gradient of a plane max goes in full to
EVERY element equal to it, and P = 0 or A = 0 (no present / no absent foreground class) makes the loss and the
image's whole foreground gradient NaN.  Ties are ranked in ascending pixel order here (kind="stable"); any order
within a tie group gives the same multiset of gradient values.
"""
import numpy as np

Q_FG, Q_BG = 0.996, 0.999  # pylayers.py:200, :207


def gwrp_weights(q, n):
    """(weights, Z) as the reference builds them (:202-203): weights[i] = q ** (n-1-i), the largest value gets 1."""
    w = np.array([q ** i for i in range(n - 1, -1, -1)])
    return w, np.sum(w)


def seed_loss(probs, labels, dtype=np.float64):
    """-mean_n( sum lab log p / sum lab ) (:104-105); NaN for an image without seeds."""
    p, l = np.asarray(probs, dtype), np.asarray(labels, dtype)
    count = l.sum(axis=(1, 2, 3), keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(-np.mean((l * np.log(p)).sum(axis=(1, 2, 3), keepdims=True) / count))


def seed_loss_grad(probs, labels, dtype=np.float64, n_global=None):
    """d loss / d probs = -lab / (p * count * N) (:108)."""
    p, l = np.asarray(probs, dtype), np.asarray(labels, dtype)
    n = n_global or p.shape[0]
    count = l.sum(axis=(1, 2, 3), keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        return l * (-1.0 / (n * count)) / p


def _parts(probs, labels, q_fg, q_bg, dtype):
    p = np.asarray(probs, dtype)
    N, M, H, W = p.shape
    n = H * W
    s = (np.asarray(labels).reshape(N, -1)[:, 1:M] > 0.5).astype(dtype)        # stat_2d (:214)
    P = s.sum(1)
    A = (M - 1) - P
    fg = p[:, 1:].reshape(N, M - 1, n)
    bg = p[:, 0].reshape(N, n)
    wf, zf = gwrp_weights(q_fg, n)
    wb, zb = gwrp_weights(q_bg, n)
    G = np.sum(np.sort(fg, axis=2) * wf / zf, axis=2)                           # probs_mean (:205)
    Gb = np.sum(np.sort(bg, axis=1) * wb / zb, axis=1)                          # probs_bg_mean (:212)
    mx = fg.max(axis=2)                                                         # probs_max (:198)
    return dict(N=N, M=M, n=n, s=s, P=P, A=A, fg=fg, bg=bg, wf=wf, zf=zf, wb=wb, zb=zb, G=G, Gb=Gb, mx=mx)


def expand_loss_terms(probs, labels, q_fg=Q_FG, q_bg=Q_BG, dtype=np.float64):
    """(loss_1, loss_2, loss_3) of :216-218."""
    d = _parts(probs, labels, q_fg, q_bg, dtype)
    s, P, A = d["s"], d["P"][:, None], d["A"][:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        l1 = -np.mean(np.sum(s * np.log(d["G"]) / P, axis=1))
        l2 = -np.mean(np.sum((1 - s) * np.log(1 - d["mx"]) / A, axis=1))
    l3 = -np.mean(np.log(d["Gb"]))
    return float(l1), float(l2), float(l3)


def expand_loss(probs, labels, q_fg=Q_FG, q_bg=Q_BG, dtype=np.float64):
    """loss_1 + loss_2 + loss_3 (:220)."""
    return sum(expand_loss_terms(probs, labels, q_fg, q_bg, dtype))


def expand_loss_grad(probs, labels, q_fg=Q_FG, q_bg=Q_BG, dtype=np.float64, n_global=None):
    """d loss / d probs (:223): through the sort permutation (rank i gets coef * w_i / Z) and, for the foreground,
    the full max term on every element equal to the plane max (eq(xmax, x) * g_max: 0 * NaN stays NaN)."""
    d = _parts(probs, labels, q_fg, q_bg, dtype)
    N, M, n = d["N"], d["M"], d["n"]
    inv = 1.0 / (n_global or N)
    with np.errstate(divide="ignore", invalid="ignore"):
        cs = -inv * (d["s"] / d["P"][:, None]) / d["G"]                         # d loss / d G_fg
        cm = inv * ((1 - d["s"]) / d["A"][:, None]) / (1 - d["mx"])              # d loss / d max
        g_fg = np.empty((N, M - 1, n), dtype)
        np.put_along_axis(g_fg, np.argsort(d["fg"], axis=2, kind="stable"), cs[..., None] * (d["wf"] / d["zf"]),
                          axis=2)
        g_fg = g_fg + (d["fg"] == d["mx"][..., None]) * cm[..., None]
    g_bg = np.empty((N, n), dtype)
    np.put_along_axis(g_bg, np.argsort(d["bg"], axis=1, kind="stable"),
                      (-inv / d["Gb"])[:, None] * (d["wb"] / d["zb"]), axis=1)
    shape = np.asarray(probs).shape
    return np.concatenate([g_bg.reshape(N, 1, n), g_fg], axis=1).reshape(shape)


def tie_canonical(grad, probs):
    """Gradient values sorted within every group of equal input values of a plane: the device and Theano may rank
    tied elements differently, and any such order gives the same sorted values."""
    g = np.asarray(grad, np.float64).reshape(-1, np.asarray(probs)[0, 0].size)
    x = np.asarray(probs, np.float64).reshape(g.shape)
    out = np.empty_like(g)
    for r in range(g.shape[0]):
        order = np.lexsort((np.nan_to_num(g[r], nan=np.inf), x[r]))
        out[r] = g[r][order]
    return out
