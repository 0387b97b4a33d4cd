"""High-precision references and error bars for the pinball loss (``pert_pinball_loss``), the eval metrics
(``pert_eval_metrics``) and the Adam step (``pert_adam_step`` and its data-parallel form ``pert_allreduce_adam``).

Every reference takes its inputs as the C ABI receives them: ``y`` int64, ``yhat`` / ``p`` / ``g`` / ``m`` / ``v``
float32, and the hyperparameters (tau, lr, beta1, beta2, eps, weight_decay, grad_scale) rounded to float32.  u = 2^-24
is the unit roundoff of float32.  Each bar is derived from the operations the kernel performs; the derivation sits next
to the bar.  ``*_f32`` are numpy float32 restatements of the kernels, with switches for the defects the bars must catch
(tests/test_loss_adam_ref.py)."""
import math

import numpy as np

U = 2.0 ** -24          # float32 unit roundoff
U64 = 2.0 ** -53        # float64 unit roundoff
F32 = np.float32


def f32(x):
    """A Python float as the C ABI's float argument receives it."""
    return float(F32(x))


# ---------------------------------------------------------------------------------------------------- pinball loss
def pinball_ref(y, yhat, tau, grad_scale=1.0, live=None):
    """Loss over the live graphs and dloss/dyhat [B], in fp64 on float32(y) and yhat.  ``live``: the live count of a
    padded batch (clamped to B, as the kernel clamps live[1]); the ghosts above it get dyhat = 0 exactly.  A tie (e = 0)
    gets torch.maximum's even split 0.5 * (1 - 2 tau)."""
    tau, gs = f32(tau), f32(grad_scale)
    B = len(y)
    bl = B if live is None else min(B, int(live))
    yf = np.asarray(y[:bl]).astype(np.float32).astype(np.float64)
    e = yf - np.asarray(yhat[:bl], dtype=np.float32).astype(np.float64)
    loss = math.fsum(np.maximum(tau * e, (tau - 1.0) * e).tolist()) / bl
    d = np.where(e > 0, -tau, np.where(e < 0, 1.0 - tau, 0.5 * (1.0 - 2.0 * tau)))
    dyhat = np.zeros(B)
    dyhat[:bl] = gs * d / bl
    return loss, dyhat


def pinball_loss_bar(bl):
    """Relative bar of the loss over ``bl`` live graphs.  Every term max(tau e, (tau-1) e) is >= 0, so no sum cancels and
    each rounding costs at most u of the total: a term rounds e = y - yhat, tau - 1 and the product (3u); one thread of
    the single 256-thread block adds ceil(bl/256) terms in sequence (ceil(bl/256) - 1), the warp shuffle tree and the
    tree over the 8 warp partials have 5 levels each (10), and the mean divides once (1): (ceil(bl/256) + 13) u."""
    return (math.ceil(bl / 256) + 13) * U


# dyhat = grad_scale * d / bl with d one of -tau (exact), 1 - tau (1 rounding) or 0.5 * (1 - 2 tau) (2 tau and the
# halving are exact, 1 - 2 tau rounds once); the product and the quotient round once each (bl < 2^24 converts
# exactly): 3u of |dyhat|, bar 4u.  A zero reference (tau = 0, tau = 1, a tie at tau = 0.5) must come out exactly 0.
PINBALL_DYHAT_BAR = 4 * U


def pinball_f32(y, yhat, tau, grad_scale=1.0, live=None, defect=None):
    """float32 restatement of k_pinball: per-thread strided sums over 256 lanes, a tree over the lanes, the mean.
    defect: 'capacity' divides by B instead of the live count; 'tie0' / 'tie_neg_tau' give a tie the gradient 0 / -tau."""
    tau, gs = F32(tau), F32(grad_scale)
    B = len(y)
    bl = B if live is None else min(B, int(live))
    e = np.asarray(y[:bl]).astype(np.float32) - np.asarray(yhat[:bl], dtype=np.float32)
    a, b = tau * e, (tau - F32(1)) * e
    terms = np.maximum(a, b)
    lanes = np.zeros(-(-bl // 256) * 256, np.float32)
    lanes[:bl] = terms
    part = lanes.reshape(-1, 256)
    s = part[0].copy()
    for row in part[1:]:
        s = s + row
    while s.size > 1:
        s = s[: s.size // 2] + s[s.size // 2:]
    den = F32(B if defect == "capacity" else bl)
    loss = float(s[0] / den)
    tie = {"tie0": F32(0), "tie_neg_tau": -tau}.get(defect, F32(0.5) * (F32(1) - F32(2) * tau))
    d = np.where(a > b, -tau, np.where(a < b, F32(1) - tau, tie)).astype(np.float32)
    dyhat = np.zeros(B, np.float32)
    dyhat[:bl] = gs * d / den
    return loss, dyhat


def pinball_worst(loss, dyhat, ref_loss, ref_dyhat, bl):
    """Largest error of (loss, dyhat) as a fraction of its bar (<= 1 passes); a nonzero dyhat where the reference is 0
    counts as infinitely far."""
    rl = abs(loss - ref_loss) / (pinball_loss_bar(bl) * abs(ref_loss)) if ref_loss != 0 else (0.0 if loss == 0 else
                                                                                              math.inf)
    dyhat = np.asarray(dyhat, dtype=np.float64)
    err = np.abs(dyhat - ref_dyhat)
    bar = PINBALL_DYHAT_BAR * np.abs(ref_dyhat)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bar > 0, err / np.where(bar > 0, bar, 1.0), np.where(err == 0, 0.0, np.inf))
    return rl, float(r.max()) if r.size else 0.0


# ---------------------------------------------------------------------------------------------------- eval metrics
def metrics_terms(y, yhat, tau):
    """The three per-graph terms exactly as k_eval_metrics forms them: correctly rounded float32 operations on
    yt = float32(y) (the reference's y.float() promotion): |yhat - yt|, that over yt, max(tau e, (tau - 1) e) with
    e = yt - yhat.  The build has no fast-math, so the kernel's division is IEEE and every term matches bit for bit."""
    tau = F32(tau)
    yt = np.asarray(y).astype(np.float32)
    yhat = np.asarray(yhat, dtype=np.float32)
    e = yt - yhat
    ae = np.abs(yhat - yt)
    return ae, ae / yt, np.maximum(tau * e, (tau - F32(1)) * e)


def metrics_ref(y, yhat, tau):
    """(sum |yhat - y|, sum |yhat - y| / y, sum of the pinball terms), each an exactly rounded sum (math.fsum) of the
    float32 terms of ``metrics_terms``."""
    return tuple(math.fsum(t.astype(np.float64).tolist()) for t in metrics_terms(y, yhat, tau))


def metrics_bar(n_terms):
    """Relative bar of one accumulator after adding ``n_terms`` terms, in any number of calls.  The terms are exact
    and >= 0 (y >= 1), so only the double additions round, each by at most 2^-53 of the total, and no term passes
    through more than n_terms - 1 of them (an addition of 0 is exact): n_terms * 2^-53."""
    return max(n_terms, 1) * U64


def metrics_f64_terms(y, yhat, tau):
    """A defective restatement: the terms in double on the exact int64 y instead of the float32 promotion."""
    tau = f32(tau)
    yd = np.asarray(y).astype(np.float64)
    yh = np.asarray(yhat, dtype=np.float32).astype(np.float64)
    e = yd - yh
    ae = np.abs(yh - yd)
    return ae, ae / yd, np.maximum(tau * e, (tau - 1.0) * e)


# ---------------------------------------------------------------------------------------------------- Adam
def adam_hyper(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, grad_scale=1.0):
    """Hyperparameters as the C ABI receives them (float32)."""
    return dict(lr=f32(lr), b1=f32(betas[0]), b2=f32(betas[1]), eps=f32(eps), wd=f32(weight_decay),
                gs=f32(grad_scale))


def adam_ref(p, g, m, v, step, hp):
    """One step of torch.optim.Adam's definition in fp64 from the float32 state (p, g, m, v): L2 weight decay added to
    the scaled gradient, m by lerp, bias corrections 1 - beta^t in double.  Returns (p, m, v) in float64."""
    p, g, m, v = (np.asarray(a, dtype=np.float32).astype(np.float64) for a in (p, g, m, v))
    gi = g * hp["gs"]
    if hp["wd"] != 0.0:
        gi = gi + hp["wd"] * p
    m1 = m + (1.0 - hp["b1"]) * (gi - m)
    v1 = hp["b2"] * v + (1.0 - hp["b2"]) * gi * gi
    bc1 = 1.0 - hp["b1"] ** step
    c2 = math.sqrt(1.0 - hp["b2"] ** step)
    p1 = p - (hp["lr"] / bc1) * (m1 / (np.sqrt(v1) / c2 + hp["eps"]))
    return p1, m1, v1


def adam_bars(p, g, m, v, step, hp, ref):
    """Absolute bars of (m, v, delta = p_new - p) for one kernel step from the float32 state (p, g, m, v), ``ref`` =
    adam_ref of that state.  G = |g gs| + |wd p| bounds the scaled, decayed gradient gi.

    gi: the product and the weight-decay fma round once each, |dgi| <= 2u G.
    m = m + (1 - b1)(gi - m) (1 - b1 is exact for b1 >= 0.5): the difference, product and sum round once each, with
        (1 - b1) <= 1/2 at most 2.5u (|m| + G) together with dgi; bar 4u (|m| + G).  The scale is |m| + G and not |m_new|
        because the lerp can cancel.
    v = b2 v + (1 - b2) gi^2: all terms >= 0; three roundings (3u v_new) plus 2 (1 - b2)|gi||dgi| <= 4u (1 - b2) G^2;
        bar 8u (b2 v + (1 - b2) G^2).
    delta = -S m_new / D, S = lr / bc1 and c2 = sqrt(bc2) each rounded once to float, D = sqrt(v_new) / c2 + eps: sqrt,
        the two quotients and the sum round once each (with S, c2: 6u |delta|), bar 8u |delta|; plus what the kernel's own
        m_new and v_new carry in, S / D * bar_m and |delta| / D * bar_v / (2 c2 sqrt(v_new)) to first order; plus one
        ulp of p_new for the final rounding of p + delta."""
    p, g, m, v = (np.asarray(a, dtype=np.float32).astype(np.float64) for a in (p, g, m, v))
    p1, m1, v1 = ref
    G = np.abs(g * hp["gs"]) + np.abs(hp["wd"] * p)
    bar_m = 4 * U * (np.abs(m) + G)
    bar_v = 8 * U * (hp["b2"] * v + (1.0 - hp["b2"]) * G * G)
    S = hp["lr"] / (1.0 - hp["b1"] ** step)
    c2 = math.sqrt(1.0 - hp["b2"] ** step)
    sq = np.sqrt(v1)
    D = sq / c2 + hp["eps"]
    delta = p1 - p
    with np.errstate(divide="ignore", invalid="ignore"):
        from_v = np.where(sq > 0, np.abs(delta) / D * bar_v / (2 * c2 * np.where(sq > 0, sq, 1.0)), 0.0)
    ulp_p = np.spacing(np.abs(p1).astype(np.float32)).astype(np.float64)
    bar_d = 8 * U * np.abs(delta) + S / D * bar_m + from_v + ulp_p
    return bar_m, bar_v, bar_d


def adam_worst(p, g, m, v, step, hp, out):
    """Largest error of the kernel's (p_new, m_new, v_new) = ``out`` as a fraction of each bar: (m, v, delta)."""
    ref = adam_ref(p, g, m, v, step, hp)
    bar_m, bar_v, bar_d = adam_bars(p, g, m, v, step, hp, ref)
    p0 = np.asarray(p, dtype=np.float32).astype(np.float64)
    pk, mk, vk = (np.asarray(a, dtype=np.float32).astype(np.float64) for a in out)

    def worst(err, bar):
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(bar > 0, err / np.where(bar > 0, bar, 1.0), np.where(err == 0, 0.0, np.inf))
        return float(r.max()) if r.size else 0.0

    return (worst(np.abs(mk - ref[1]), bar_m), worst(np.abs(vk - ref[2]), bar_v),
            worst(np.abs((pk - p0) - (ref[0] - p0)), bar_d))


def adam_f32(p, g, m, v, step, hp, defect=None):
    """float32 restatement of the kernel (corrections from double, as the library now computes them).  defect:
    'bc_off_by_one' uses step + 1 in both corrections; 'adamw' decays p by lr wd instead of adding wd p to the gradient;
    'eps_in_sqrt' takes sqrt(v / bc2 + eps); 'fp32_bc' forms 1 - beta^t, its square root and lr / bc1 in float32."""
    p, g, m, v = (np.asarray(a, dtype=np.float32) for a in (p, g, m, v))
    lr, b1, b2, eps, wd, gs = (F32(hp[k]) for k in ("lr", "b1", "b2", "eps", "wd", "gs"))
    one = F32(1)
    gi = g * gs
    if wd != 0 and defect != "adamw":
        gi = gi + wd * p
    m1 = m + (one - b1) * (gi - m)
    v1 = b2 * v + (one - b2) * gi * gi
    t = step + 1 if defect == "bc_off_by_one" else step
    if defect == "fp32_bc":
        with np.errstate(over="ignore"):
            bc1 = one - b1 ** F32(t)
            bc2 = one - b2 ** F32(t)
        S, c2 = lr / bc1, np.sqrt(bc2)
    else:
        S = F32(float(lr) / (1.0 - float(b1) ** t))
        c2 = F32(math.sqrt(1.0 - float(b2) ** t))
    if defect == "eps_in_sqrt":
        den = np.sqrt(v1 / (c2 * c2) + eps)
    else:
        den = np.sqrt(v1) / c2 + eps
    p0 = p * (one - lr * wd) if defect == "adamw" else p
    return (p0 - S * (m1 / den)).astype(np.float32), m1.astype(np.float32), v1.astype(np.float32)


def adam_state(n, seed, zero_frac=0.05):
    """Seeded float32 parameters and a gradient with magnitudes from 1e-12 to 1e3, random signs and some zeros."""
    rng = np.random.default_rng(seed)
    p = rng.standard_normal(n).astype(np.float32)
    p[rng.random(n) < zero_frac] = 0.0
    return p, adam_grad(n, rng, zero_frac)


def adam_grad(n, rng, zero_frac=0.05):
    g = (10.0 ** rng.uniform(-12, 3, n)) * np.where(rng.random(n) < 0.5, -1.0, 1.0)
    g[rng.random(n) < zero_frac] = 0.0
    return g.astype(np.float32)


# ---------------------------------------------------------------------------------------------------- test data
def loss_data(B, seed):
    """Seeded labels and predictions for the loss and metrics: y in [1, 1e7] with a share above 2^24, yhat near y with
    some negative predictions and some exact ties (yhat == float32(y))."""
    rng = np.random.default_rng(seed)
    y = np.round(10.0 ** rng.uniform(0, 7, B)).astype(np.int64)
    big = rng.random(B) < 0.05
    y[big] = rng.integers(2 ** 24 + 1, 3 * 10 ** 7, int(big.sum()))
    yhat = (y * (1.0 + 0.3 * rng.standard_normal(B))).astype(np.float32)
    neg = rng.random(B) < 0.05
    yhat[neg] = -np.abs(yhat[neg])
    tie = rng.random(B) < 0.1
    if B >= 3:
        tie[:2] = True
    yhat[tie] = y[tie].astype(np.float32)
    return y, yhat
