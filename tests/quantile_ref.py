"""High-precision references and error bars for a global head with T quantile outputs: the head kernels at T outputs
(``k_head_fwd`` / ``k_head_bwd`` through ``pert_model_forward_q`` / ``_backward_q``), the pinball loss over [B, T]
(``pert_pinball_loss_q``) and the per-level eval metrics (``pert_eval_metrics_q``).

They extend tests/engine_parts_ref.py and tests/loss_adam_ref.py, whose conventions they keep: inputs as the kernels
receive them (float32, the engine's Hp-wide layout), fp64 results, u = 2^-24 and gamma(n) = n u / (1 - n u), and every bar
a worst-case bound derived next to it.  ``*_f32`` are numpy float32 restatements of the kernels' orders, with switches
for the defects the bars must catch (tests/test_quantile_args.py)."""
import math

import numpy as np
import torch

from tests.engine_parts_ref import HEAD_G, U, _mat, _pad, gamma, head_params

F32 = np.float32


def f32(x):
    return float(F32(x))


# ------------------------------------------------------------------------------------------------------ head
def head_params_q(d, Hp, flat, T):
    """(W1 [Hp, 2Hp], b1 [Hp], W2 [T, Hp], b2 [T], entry table [n_entry, Hp]) as k_head_* read them at T outputs."""
    W1, b1, _, _, ent = head_params(d, Hp, flat)
    W2 = _pad(_mat(flat, d.off_g2_w, T, d.H), (T, Hp))
    return W1, b1, W2, flat[d.off_g2_b:d.off_g2_b + T].clone(), ent


def head_fwd_ref_q(h1, W2, b2):
    """pred [B, T] = h1 W2^T + b2 on the kernel's own h1 (workspace code 1).  Lane j keeps, per level, the FMA chain
    over n = j, j + 32, ... (ceil(Hp / 32) roundings), a 5-step shuffle tree adds the lanes and b2[t] comes last: the
    one-output bar per level, gamma(ceil(Hp / 32) + 6) (|h1| |W2[t]| + |b2[t]|)."""
    Hp = W2.shape[1]
    h1, W2, b2 = (t.double() for t in (h1, W2, b2))
    pred = h1 @ W2.T + b2
    bar = gamma(math.ceil(Hp / 32) + 6) * (h1.abs() @ W2.abs().T + b2.abs())
    return pred, bar


def head_bwd_ref_q(dg, z, h1, W1, W2, ids, n_entry):
    """k_head_bwd at T outputs on its own inputs: dg [B, T], z, h1, W1 as in head_bwd_ref, W2 [T, Hp].
    -> dict name -> (ref, bar), float64: dpool [B, Hp], entry [n_entry, Hp], W1 [Hp, 2Hp], b1 [Hp], W2 [T, Hp], b2 [T].

    dh = sum_t dg[t] W2[t] (h1 > 0) is a product and T - 1 FMAs: T roundings of sum |dg[t]| |W2[t]| (dh_abs).  Every
    bar of the one-output head that carries the dh rounding (1 there) carries T here: dpool gamma(T + Hp / 2 + 1)
    dh_abs |W1|; an entry row gamma(T + Hp / 2 + 1 + n_r + 1); dW1 and db1 gamma(T + 8 + ceil(B / 8) + 1).  dW2[t] and
    db2[t] are level t's one-output sums: gamma(8 + ceil(B / 8) + 1) and gamma(8 + ceil(B / 8))."""
    Hp = W1.shape[0]
    B, T = dg.shape
    dg, z, h1, W1, W2 = (t.double() for t in (dg, z, h1, W1, W2))
    ids = torch.as_tensor(ids).long()
    mask = (h1 > 0).double()
    dh = (dg @ W2) * mask
    dh_abs = (dg.abs() @ W2.abs()) * mask
    dz = dh @ W1
    dz_abs = dh_abs @ W1.abs()
    n_r = torch.bincount(ids, minlength=n_entry).double()
    ent = torch.zeros(n_entry, Hp, dtype=torch.float64).index_add_(0, ids, dz[:, Hp:])
    ent_abs = torch.zeros(n_entry, Hp, dtype=torch.float64).index_add_(0, ids, dz_abs[:, Hp:])
    g_ent = (n_r + T + Hp // 2 + 2) * U
    ncta = math.ceil(B / HEAD_G)
    gw = gamma(T + HEAD_G + ncta + 1)
    return {
        "dpool": (dz[:, :Hp], gamma(T + Hp // 2 + 1) * dz_abs[:, :Hp]),
        "entry": (ent, (g_ent / (1 - g_ent))[:, None] * ent_abs),
        "W1": (dh.T @ z, gw * (dh_abs.T @ z.abs())),
        "b1": (dh.sum(0), gw * dh_abs.sum(0)),
        "W2": (dg.T @ h1, gamma(HEAD_G + ncta + 1) * (dg.abs().T @ h1.abs())),
        "b2": (dg.sum(0), gamma(HEAD_G + ncta) * dg.abs().sum(0)),
    }


def head_fwd_f32(h1, W2, b2, defect=None):
    """float32 restatement of k_head_fwd's output at T levels: per lane and level an FMA chain over n = lane + 32 k,
    a butterfly over the 32 lanes, + b2[t].  defect: 'row0' reads W2[0] for every level, 'bias0' adds b2[0] to every
    level, 'stride1' reads level t's row at offset t (rows of 1 float instead of Hp)."""
    h1 = np.asarray(h1, np.float32)
    W2 = np.asarray(W2, np.float32)
    b2 = np.asarray(b2, np.float32)
    B, Hp = h1.shape
    T = W2.shape[0]
    flatW = W2.reshape(-1)
    out = np.zeros((B, T), np.float32)
    for t in range(T):
        if defect == "row0":
            w = W2[0]
        elif defect == "stride1":
            w = flatW[t:t + Hp]
        else:
            w = W2[t]
        lanes = np.zeros((B, 32), np.float32)
        for n0 in range(0, Hp, 32):
            seg = slice(n0, min(Hp, n0 + 32))
            k = seg.stop - seg.start
            lanes[:, :k] = (h1[:, seg] * w[seg] + lanes[:, :k]).astype(np.float32)   # fmaf ~ round once
        s = lanes
        while s.shape[1] > 1:
            s = (s[:, : s.shape[1] // 2] + s[:, s.shape[1] // 2:]).astype(np.float32)
        out[:, t] = s[:, 0] + (b2[0] if defect == "bias0" else b2[t])
    return out


# ------------------------------------------------------------------------------------------------------ pinball
def pinball_q_ref(y, yhat, taus, grad_scale=1.0, live=None):
    """Loss over the live graphs' B_l T terms and dloss/dyhat [B, T] in fp64 on float32(y), yhat [B, T] and the levels
    rounded to float32; ghost rows get 0 exactly; a tie gets torch.maximum's even split 0.5 (1 - 2 tau)."""
    taus = np.array([f32(t) for t in taus])
    gs = f32(grad_scale)
    yhat = np.asarray(yhat, np.float32)
    B, T = yhat.shape
    bl = B if live is None else min(B, int(live))
    yf = np.asarray(y[:bl]).astype(np.float32).astype(np.float64)[:, None]
    e = yf - yhat[:bl].astype(np.float64)
    terms = np.maximum(taus * e, (taus - 1.0) * e)
    n = bl * T
    loss = math.fsum(terms.reshape(-1).tolist()) / n
    d = np.where(e > 0, -taus, np.where(e < 0, 1.0 - taus, 0.5 * (1.0 - 2.0 * taus)))
    dyhat = np.zeros((B, T))
    dyhat[:bl] = gs * d / n
    return loss, dyhat


def pinball_q_loss_bar(n_terms):
    """Relative bar of the loss over n_terms = B_l T terms: the single 256-thread block adds ceil(n / 256) terms per
    thread, so the one-level derivation (tests/loss_adam_ref.py pinball_loss_bar) holds with n_terms for B_l:
    (ceil(n / 256) + 13) u (B_l T < 2^24 converts exactly)."""
    return (math.ceil(n_terms / 256) + 13) * U


# dyhat = grad_scale * d / (B_l T): the one-level derivation, bar 4u of |dyhat|; a zero reference must be exactly 0
PINBALL_Q_DYHAT_BAR = 4 * U


def pinball_q_f32(y, yhat, taus, grad_scale=1.0, live=None, defect=None):
    """float32 restatement of k_pinball_q: element i = b T + t, thread i mod 256 adds its elements in order, a tree over
    the 256 lanes, the mean over B_l T.  defect: 'per_graph' divides by B_l (the one-level mean), 'level0' uses tau_0
    for every column."""
    taus = np.array([F32(t) for t in taus], np.float32)
    gs = F32(grad_scale)
    yhat = np.asarray(yhat, np.float32)
    B, T = yhat.shape
    bl = B if live is None else min(B, int(live))
    tt = np.broadcast_to(taus[:1] if defect == "level0" else taus, (bl, T))
    e = np.asarray(y[:bl]).astype(np.float32)[:, None] - yhat[:bl]
    a, c = tt * e, (tt - F32(1)) * e
    terms = np.maximum(a, c).reshape(-1)
    n = bl * T
    lanes = np.zeros(-(-n // 256) * 256, np.float32)
    lanes[:n] = terms
    part = lanes.reshape(-1, 256)
    s = part[0].copy()
    for row in part[1:]:
        s = s + row
    while s.size > 1:
        s = s[: s.size // 2] + s[s.size // 2:]
    den = F32(bl if defect == "per_graph" else n)
    d = np.where(a > c, -tt, np.where(a < c, F32(1) - tt, F32(0.5) * (F32(1) - F32(2) * tt))).astype(np.float32)
    dyhat = np.zeros((B, T), np.float32)
    dyhat[:bl] = gs * d / den
    return float(s[0] / den), dyhat


def pinball_q_worst(loss, dyhat, ref_loss, ref_dyhat, n_terms):
    """Largest error of (loss, dyhat) as a fraction of its bar (<= 1 passes)."""
    rl = abs(loss - ref_loss) / (pinball_q_loss_bar(n_terms) * abs(ref_loss)) if ref_loss != 0 else \
        (0.0 if loss == 0 else math.inf)
    dyhat = np.asarray(dyhat, dtype=np.float64)
    err = np.abs(dyhat - ref_dyhat)
    bar = PINBALL_Q_DYHAT_BAR * np.abs(ref_dyhat)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bar > 0, err / np.where(bar > 0, bar, 1.0), np.where(err == 0, 0.0, np.inf))
    return rl, float(r.max()) if r.size else 0.0


# ------------------------------------------------------------------------------------------------------ metrics
def metrics_q_ref(y, yhat, taus):
    """float64 [4T + 1] as pert_eval_metrics_q accumulates it: per level the exactly rounded sums (math.fsum) of the
    float32 terms |yhat_t - yt|, that over yt and max(tau e, (tau - 1) e) (yt = float32(y), e = yt - yhat_t), the count
    of y <= yhat_t in float32, then the count of rows with yhat_t > yhat_{t+1} for some t.  Counts are exact."""
    yhat = np.asarray(yhat, np.float32)
    B, T = yhat.shape
    yt = np.asarray(y).astype(np.float32)
    out = np.zeros(4 * T + 1)
    for t in range(T):
        tau = F32(taus[t])
        e = yt - yhat[:, t]
        ae = np.abs(yhat[:, t] - yt)
        for k, term in enumerate((ae, ae / yt, np.maximum(tau * e, (tau - F32(1)) * e))):
            out[4 * t + k] = math.fsum(term.astype(np.float64).tolist())
        out[4 * t + 3] = float(np.count_nonzero(yt <= yhat[:, t]))
    out[4 * T] = float(np.count_nonzero((yhat[:, :-1] > yhat[:, 1:]).any(1))) if T > 1 else 0.0
    return out


def metrics_q_bar(n_terms):
    """Relative bar of one level sum after n_terms terms: tests/loss_adam_ref.py metrics_bar, n_terms 2^-53."""
    return max(n_terms, 1) * 2.0 ** -53


def quantile_data(B, T, seed, cross=0.05):
    """Seeded labels y [B] in [1, 1e7] and predictions [B, T] increasing along the levels except in a ``cross`` share
    of the rows (two neighbours swapped), with exact ties on y and equal neighbouring levels in a few rows."""
    rng = np.random.default_rng(seed)
    y = np.round(10.0 ** rng.uniform(0, 7, B)).astype(np.int64)
    base = y * (1.0 + 0.3 * rng.standard_normal(B))
    steps = np.cumsum(np.abs(rng.standard_normal((B, T))) * 0.05 * y[:, None], axis=1)
    yhat = (base[:, None] + steps).astype(np.float32)
    if T > 1:
        sw = np.nonzero(rng.random(B) < cross)[0]
        j = rng.integers(0, T - 1, sw.size)
        a = yhat[sw, j].copy()
        yhat[sw, j] = yhat[sw, j + 1]
        yhat[sw, j + 1] = a
        eq = np.nonzero(rng.random(B) < 0.02)[0]
        yhat[eq, 1] = yhat[eq, 0]
    tie = rng.random(B) < 0.1
    if B >= 3:
        tie[:2] = True
    col = rng.integers(0, T, B)
    yhat[tie, col[tie]] = y[tie].astype(np.float32)
    return y, yhat
