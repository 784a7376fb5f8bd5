"""NumPy float32 statement of the reference's debug checks (dca/loss.py:87-100, NB.loss with debug=True) and of the
report the loss kernels record for one batch: per term, the count of non-finite elements and the first one in
row-major order."""
import numpy as np
from scipy.special import gammaln

TERMS = ("y_pred", "t1", "t2")


def debug_terms(y, m, sf, theta):
    """y_pred, t1, t2 of every element, float32: y, m [B x G]; sf [B] (None: 1); theta broadcastable to [B x G] (per
    element, per gene [G] or per cell [B x 1])."""
    f = np.float32
    y, m = np.asarray(y, f), np.asarray(m, f)
    sf = np.ones(y.shape[0], f) if sf is None else np.asarray(sf, f)
    theta = np.broadcast_to(np.asarray(theta, f), y.shape)
    eps = f(1e-10)
    with np.errstate(all="ignore"):
        th = np.minimum(theta, f(1e6))
        yp = m * sf[:, None]
        te = th + eps
        lg = lambda v: gammaln(v).astype(f)                       # noqa: E731
        t1 = lg(te) + lg(y + f(1)) - lg(y + th + eps)
        t2 = (th + y) * np.log(f(1) + yp / te) + y * (np.log(te) - np.log(yp + eps))
    return yp, t1, t2


def debug_report(y, m, sf, theta):
    """engine.read_debug_report()'s dict for the same batch."""
    count, first = [], []
    for t in debug_terms(y, m, sf, theta):
        bad = np.argwhere(~np.isfinite(t))
        count.append(int(len(bad)))
        first.append(tuple(int(v) for v in bad[0]) if len(bad) else None)
    return {"count": count, "first": first}
