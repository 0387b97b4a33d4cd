"""-m gpu tests of the BatchNorm pieces that run inside other kernels, against float64 on the hard graphs of
tests/test_gpu_tconv_structure.py and on columns far from zero mean:

  a. the forward statistics in the epilogue of the staged conv forward (pert_tconv_fwd_stats);
  b. those statistics fed to the node-linear forward that applies BatchNorm (pert_bn_linear_fwd_planes, stats_ready);
  c. the backward column sums folded into the node-linear backward (pert_linear_bwd_planes_ex);
  d. the backward apply folded into the conv backward target pass (pert_tconv_bwd_bn);
  e. whole engine steps with shifted and constant BatchNorm inputs, against the fp64 oracle.

Every output starts filled with a sentinel; rows at or past N and the memory after each buffer must stay untouched.

u = 2^-24, u64 = 2^-53.  A sequential fp32 sum of terms t_i of depth D is off by at most D u sum |t_i| (the gamma_D
bound, D u << 1 throughout), and every further rounding adds u times the size of the value it rounds.

a. Forward statistics.  A CTA owns a tile of T consecutive nodes; its lane groups (LPR lanes per node row) take the
   nodes GPC apart (GPC = lane groups per CTA, GPW = 32 / LPR per warp): 256-thread CTAs with LPR = H/8 when two CTAs
   fit an SM, 1024-thread CTAs with LPR = H/4 otherwise.  A lane sums ceil(T / GPC) rows in fp32, a shuffle tree of
   log2(GPW) levels adds the warp's groups, shared-memory fp64 atomics add the warps.  So the tile sums have depth
   Df = ceil(T / GPC) + log2(GPW) (the larger of the two CTA shapes), and the fp32 tile mean mu_b = fl(S_b / n_b) is
   off from the exact tile mean m_b by delta_b <= (Df + 1) u mean_b|o|.  The second pass sums (o - mu_b)^2 over the
   same depths: a rounded difference and an fma per term, (Df + 3) u sum_b (o - mu_b)^2 <= (Df + 3) u (M2 + sum_b n_b
   delta_b^2).  The tiles combine as acc[c] = sum n_b mu_b, acc[H + c] = sum (M2_b + n_b mu_b^2) in fp64; the test
   takes mean = acc[c] / n and var = (acc[H + c] - n mean^2) / n as bn_batch_stats does.  Exactly (Chan's combine),
   n var = M2 + n (m - mean)^2 - 2 sum_b n_b (mu_b - mean)(m_b - mu_b) + the rounding above, so with nb tiles
     |mean - m| <= (Df + 2) u mean|o| + (nb + 2) u64 mean|o|,
     |var - v| <= [(Df + 3) u (M2 + sum n_b delta_b^2) + 2 sum n_b |m_b - m| delta_b + 3 sum n_b delta_b^2] / n
                  + (2 nb + 8) u64 mean o^2.
   These are test_gpu_nodeops' BatchNorm bars with the conv's depths instead of k_bn_partial's.  A constant column
   has o - mu_b = 0 up to the rounding of mu_b, so its variance is within (Df + 1)^2 u^2 o^2 of 0 and its rstd is
   fp32(1 / sqrt(eps)).  The raw (uncentred) sums the epilogue kept
   before are off by about Df u mean^2 / sqrt(lanes): at mean 1e3 / std 1 that is 1e-3 of the variance, tens of times
   the bar above, and a constant column got a variance of rounding noise (rstd 80-230 instead of 316).
b. The apply at the epilogue's statistics: mean / rstd / running statistics under the same bars carried through
   test_gpu_nodeops' formulas (rstd by the mean value theorem, running statistics 3 u of their terms plus momentum
   times the bar of the batch value); x[l] = relu(fma((o - mean) rstd, gamma, beta)) against fp64 of that formula at
   the kernel's own fp32 mean / rstd: 3 u (|gamma| |o - mean| rstd + |y|).
c. pert_linear_bwd_planes_ex: a thread reduces two rows of each 64-row tile of its cluster's share (ceil(tiles /
   clusters) tiles; an H100 places at least 16 clusters of four CTAs) in fp32, one shuffle adds its lane pair, the four
   warps and the CTAs add in fp64: depth Ds = 2 ceil(tiles / 16) + 1.  dz = fl(dX relu_scale) is exact data here (it
   is recomputed from the kernel's dX as the kernel rounds it), xhat = (x - mean) rstd takes two roundings and the fma
   one: Ea = Ds u sum |dz|, Eb = (Ds + 3) u sum |dz xhat|.  dX must be bit-identical to pert_linear_bwd_planes;
   dW4 / db4 keep test_gpu_linear_bwd's bars.
d. pert_tconv_bwd_bn with exact fp64 sums as input: g = gamma rstd (dz - a/n - xhat b/n) in fp32: the 8 roundings of
   pert_bn_bwd's apply (test_gpu_nodeops) plus the fp32 rounding of each fp64 sum, 10 u (|dz| + |a|/n + |xhat| |b|/n)
   times |gamma| rstd; ghost rows (>= live[0]) exactly +0.0.  dbeta = fl(dbeta0 + fl(a)): 2 u (|dbeta0| + |a|), so a
   sum added twice or not at all fails.  dq / dk / dv / ds / the table gradients against fp64 of the conv backward at
   the fp64 g, under the bars of test_gpu_tconv_structure (the fp32 g is within 1e-6 of it, an order below those).
e. One cfg2 training step per width with lin_skip biases shifted by 1e2 and one constant conv output column, against
   the fp32 / fp64 oracles (tests/helpers.py assert_close_ref), with and without dropout; one padded (bucketed) step
   against the eager step on the same model.
"""
import copy
import ctypes
import math

import numpy as np
import pytest
import torch

from tests.helpers import assert_close
from tests.test_gpu_tconv_structure import (BUILDERS, HUB_BAR, NODE_BAR, SHARP_BAR, TABLE_BAR, Graph, _ref_run,
                                            graph, make_inputs, ref_tconv, tile_geom)

pytestmark = pytest.mark.gpu

U, U64 = 2.0 ** -24, 2.0 ** -53
SENT = 12345.0
EPS = float(np.float32(1e-5))
MOM = 0.1
RSTD_CONST = float(np.float32(1.0 / math.sqrt(EPS)))   # bn_batch_stats at var = 0: (float)(1 / sqrt(0 + (double)eps))
CONST_COL, CONST_VAL = 1, 7.25
UNSUPPORTED = -2


def _L():
    from pert_gnn_kdd23_b200 import _lib

    return _lib


def _st():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return None if t is None else t.data_ptr()


def _bar_of(name):
    return {"sharp": SHARP_BAR, "in_hub": HUB_BAR, "out_hub": HUB_BAR}.get(name, NODE_BAR)


# ------------------------------------------------------------------------------------------------------ conv inputs
def _stress_inputs(g, H, n_rpc, tables):
    """make_inputs with stress columns in the conv output.  Column CONST_COL is constant on every graph (v and both
    table columns zero, so out = s there: sum alpha = 1 or no in-edges).  On the edgeless graph out = s exactly:
    column 0 has mean 1e3 / std 1 and column 2 one outlier.  On the others a quarter of the columns is shifted by 1e2
    and another quarter by 1e3."""
    q, k, v, s, t_if, t_rpc, gout = make_inputs(g, H, n_rpc, tables)
    v[:, CONST_COL] = 0.0
    if tables:
        t_if[:, CONST_COL] = 0.0
        t_rpc[:, CONST_COL] = 0.0
    s = s.clone()
    if g.E == 0:
        gen = torch.Generator().manual_seed(H)
        s[:, 0] = 1e3 + torch.randn(g.N, generator=gen)
        s[:, 2] = 0.1 * torch.randn(g.N, generator=gen)
        s[g.N // 3, 2] = 5e3
    else:
        s[:, 4::4] += 1e2
        s[:, 6::4] += 1e3
    s[:, CONST_COL] = CONST_VAL
    return q, k, v, s, t_if, t_rpc, gout


class _Conv:
    """Device operands of one graph at width H (planes q | k | v | s, index, tables)."""

    def __init__(self, g, H, n_rpc, tables, hint=True, inputs=None):
        from pert_gnn_kdd23_b200.index import build_index

        self.g, self.H, self.N, self.E = g, H, g.N, g.E
        self.n = n_rpc if tables else 0
        self.B = g.B if hint else 0
        self.cpu = inputs if inputs is not None else _stress_inputs(g, H, n_rpc, tables)
        q, k, v, s, t_if, t_rpc, _ = self.cpu
        ei = torch.from_numpy(np.stack([g.src, g.dst])).cuda()
        ea = torch.from_numpy(np.stack([g.if_id, g.rpc_id(max(n_rpc, 1))], 1)).cuda() if tables else None
        self.gi = build_index(ei, g.N, ea, g.n_if if tables else 0, n_rpc if tables else 0).check()
        self.pl = torch.stack([q, k, v, s]).cuda().contiguous()
        self.t_if = t_if.cuda().contiguous() if tables else None
        self.t_rpc = t_rpc.cuda().contiguous() if tables else None
        self.csr_if = self.gi.csr_if if tables else None
        self.csr_rpc = self.gi.csr_rpc if tables else None

    def fwd_args(self, out, alpha):
        gi, pl = self.gi, self.pl
        return (_ptr(pl[0]), _ptr(pl[1]), _ptr(pl[2]), _ptr(pl[3]), self.H, _ptr(gi.rowptr), _ptr(gi.csr_src),
                _ptr(self.csr_if), _ptr(self.csr_rpc), _ptr(self.t_if), _ptr(self.t_rpc), _ptr(out), self.H,
                _ptr(alpha), self.n, self.N, self.E, self.B, self.H, self.H)

    def forward(self, live=None, stats=True):
        """-> (out buffer [(N + 2) H + 64] with sentinels after the rows, alpha, acc buffer [2H + 16] or None)."""
        L, H, N = _L(), self.H, self.N
        out = torch.full(((N + 2) * H + 64,), SENT, device="cuda")
        alpha = torch.full((max(self.E, 1),), float("nan"), device="cuda")
        if not stats:
            L.call("pert_tconv_fwd_c", *self.fwd_args(out, alpha), _st())
            return out, alpha, None
        acc = torch.full((2 * H + 16,), SENT, dtype=torch.float64, device="cuda")
        acc[:2 * H] = 0.0
        fused = ctypes.c_int(-1)
        L.call("pert_tconv_fwd_stats", *self.fwd_args(out, alpha), _ptr(acc), _ptr(live), ctypes.byref(fused), _st())
        torch.cuda.synchronize()
        assert fused.value == 1, "the staged tile kernel should take every shape here"
        return out, alpha, acc


def _tile_depth(H, T):
    """Df of the module docstring: the deeper of the two CTA shapes."""
    d = 0
    for nt, lpr in ((256, H // 8), (1024, H // 4)):
        gpc, gpw = nt // lpr, 32 // lpr
        d = max(d, math.ceil(T / gpc) + int(math.log2(gpw)))
    return d


def _stat_ref(o64, T, Df):
    """fp64 mean / biased variance of the rows o64 [n, H] and the bars of part a (tiles of T rows)."""
    n, H = o64.shape
    m = o64.mean(0)
    M2 = ((o64 - m) ** 2).sum(0)
    nb = math.ceil(n / T)
    pad = nb * T - n
    op = torch.nn.functional.pad(o64, (0, 0, 0, pad)).view(nb, T, H)
    n_b = torch.full((nb, 1), float(T), dtype=torch.float64, device=o64.device)
    n_b[-1] = T - pad
    m_b = op.sum(1) / n_b
    delta = (Df + 1) * U * op.abs().sum(1) / n_b
    absm = o64.abs().mean(0)
    Em = (Df + 2) * U * absm + (nb + 2) * U64 * absm
    Evar = ((Df + 3) * U * (M2 + (n_b * delta ** 2).sum(0)) + (2 * n_b * (m_b - m).abs() * delta).sum(0)
            + (3 * n_b * delta ** 2).sum(0)) / n + (2 * nb + 8) * U64 * (o64 * o64).mean(0)
    return m, M2 / n, Em, Evar


def _ratio(got, ref, bar):
    err = (got.double() - ref.double()).abs()
    return float((err / bar.clamp_min(1e-300)).max()) if err.numel() else 0.0


def _assert_bar(got, ref, bar, what):
    r = _ratio(got, ref, bar)
    assert r <= 1.0, f"{what}: element-wise error {r:.3g} x the bar"


# ------------------------------------------------------------------------------------------------------ a + b
def _live_values(g, H, n, hint=True):
    T = tile_geom(H, n, g.N, g.E, g.B if hint else 0)[0]
    vals = [None, g.N, g.N - 1, 1]
    vals += [v for v in (T - 1, T + 1) if 1 <= v < g.N]
    return T, vals


def _check_stats(c, out, acc, live_val, T, tag):
    H, N = c.H, c.N
    o = out[:N * H].view(N, H)
    assert bool((out[N * H:] == SENT).all()), f"out past row N written ({tag})"
    assert bool((acc[2 * H:] == SENT).all()), f"memory after bn_acc written ({tag})"
    n = N if live_val is None else min(live_val, N)
    o64 = o[:n].double()
    m, v, Em, Evar = _stat_ref(o64, T, _tile_depth(H, T))
    a = acc[:2 * H]
    mean = a[:H] / n
    var = (a[H:] - n * mean * mean).clamp_min(0) / n
    _assert_bar(mean, m, Em, f"mean ({tag})")
    _assert_bar(var, v, Evar, f"variance ({tag})")
    rs = float(np.float32(1.0 / math.sqrt(float(var[CONST_COL]) + EPS)))
    assert rs == RSTD_CONST, f"constant column: rstd {rs} ({tag})"
    return mean, var


def _apply_check(c, out, acc, tag):
    """Part b: acc as the workspace of pert_bn_linear_fwd_planes with stats_ready = 1."""
    L, H, N = _L(), c.H, c.N
    o = out[:N * H].view(N, H)
    gen = torch.Generator().manual_seed(N + H)
    gamma, beta = (1 + 0.3 * torch.randn(H, generator=gen)).cuda(), (0.2 * torch.randn(H, generator=gen)).cuda()
    rm0, rv0 = (0.1 * torch.randn(H, generator=gen)).cuda(), (1 + torch.rand(H, generator=gen)).cuda()
    rm, rv = rm0.clone(), rv0.clone()
    nbt = torch.tensor([3], dtype=torch.int64, device="cuda")
    W4 = (torch.randn(4 * H, H, generator=gen) / math.sqrt(H)).cuda()
    b4 = (0.1 * torch.randn(4 * H, generator=gen)).cuda()
    mean = torch.full((H + 4,), SENT, device="cuda")
    rstd = torch.full((H + 4,), SENT, device="cuda")
    x_out = torch.full((N * H + 64,), SENT, device="cuda")
    planes = torch.empty(4 * N * H, device="cuda")
    ws = acc.clone()
    ws_bytes = L.lib().pert_bn_workspace_bytes(N, H)
    assert ws.numel() * 8 >= 2 * H * 8
    L.call("pert_bn_linear_fwd_planes", _ptr(o), H, 1, _ptr(gamma), _ptr(beta), _ptr(rm), _ptr(rv), _ptr(nbt), EPS,
           MOM, 1, _ptr(mean), _ptr(rstd), _ptr(x_out), H, _ptr(ws), ws_bytes, 1, 0.0, None, 0, _ptr(W4), H,
           _ptr(b4), _ptr(planes), N * H, N, H, H, _st())
    torch.cuda.synchronize()
    T = tile_geom(H, c.n, N, c.E, c.B)[0]
    m, v, Em, Evar = _stat_ref(o.double(), T, _tile_depth(H, T))
    _assert_bar(mean[:H], m, Em + U * m.abs(), f"apply mean ({tag})")
    r = 1.0 / torch.sqrt(v + EPS)
    Ers = 0.5 * Evar * (v + EPS - Evar).clamp_min(EPS) ** -1.5 + 2 * U * r
    _assert_bar(rstd[:H], r, Ers, f"apply rstd ({tag})")
    assert float(rstd[CONST_COL]) == RSTD_CONST, f"constant column rstd {float(rstd[CONST_COL])} ({tag})"
    assert bool((mean[H:] == SENT).all()) and bool((rstd[H:] == SENT).all()), f"mean / rstd past H ({tag})"
    mom = float(np.float32(MOM))
    rm_ref = (1 - mom) * rm0.double() + mom * m
    _assert_bar(rm, rm_ref, 3 * U * ((1 - mom) * rm0.double().abs() + mom * m.abs()) + mom * Em, f"running_mean ({tag})")
    k = N / (N - 1)
    rv_ref = (1 - mom) * rv0.double() + mom * v * k
    _assert_bar(rv, rv_ref, 3 * U * ((1 - mom) * rv0.double().abs() + mom * v * k) + mom * (Evar * k + U * v * k),
                f"running_var ({tag})")
    assert int(nbt) == 4, f"num_batches_tracked ({tag})"
    m_k, rs_k, ga, be = mean[:H].double(), rstd[:H].double(), gamma.double(), beta.double()
    d = o.double() - m_k
    y_ref = d * rs_k * ga + be
    bar = 3 * U * (ga.abs() * d.abs() * rs_k + y_ref.abs())
    _assert_bar(x_out[:N * H].view(N, H), y_ref.clamp_min(0), bar, f"x[l] ({tag})")
    assert bool((x_out[N * H:] == SENT).all()), f"memory after x[l] written ({tag})"


@pytest.mark.parametrize("H", [32, 64, 128])
@pytest.mark.parametrize("name", list(BUILDERS))
def test_forward_statistics(name, H):
    """pert_tconv_fwd_stats on every builder (big_graph runs whole-SM tiles at every width, the others at H = 128):
    out bit-identical to pert_tconv_fwd_c, the statistics of the rows below live[0] within the centred bars; at H = 64
    and N >= 4096 the statistics also feed the BatchNorm apply of the node-linear forward (part b)."""
    g = graph(name)
    c = _Conv(g, H, 8, True)
    ref_out, ref_alpha, _ = c.forward(stats=False)
    T, lives = _live_values(g, H, c.n)
    for lv in lives:
        live = None if lv is None else torch.tensor([lv, g.B], dtype=torch.int64, device="cuda")
        out, alpha, acc = c.forward(live)
        tag = f"{name} H={H} live={lv}"
        assert torch.equal(out, ref_out), f"out differs from pert_tconv_fwd_c ({tag})"
        assert torch.equal(alpha[:g.E], ref_alpha[:g.E]), f"alpha differs from pert_tconv_fwd_c ({tag})"
        _check_stats(c, out, acc, lv, T, tag)
        if lv is None and H == 64 and g.N >= 4096:
            _apply_check(c, out, acc, tag)


@pytest.mark.parametrize("variant", ["no_tables", "rpc1", "no_hint", "one_node", "live_past_n"])
@pytest.mark.parametrize("H", [32, 64, 128])
def test_forward_statistics_variants(H, variant):
    """No edge tables, one rpc type and a zero size hint (other tile sizes) on the dense graph; a one-node batch (its
    tile is smaller than the epilogue's scratch); live[0] > N counts every row."""
    name = "dense"
    if variant == "one_node":
        g = Graph([1], np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0))
    else:
        g = graph(name)
    kw = {"no_tables": dict(tables=False), "rpc1": dict(n_rpc=1), "no_hint": dict(hint=False)}.get(variant, {})
    c = _Conv(g, H, kw.get("n_rpc", 8), kw.get("tables", True), kw.get("hint", True))
    ref_out, _, _ = c.forward(stats=False)
    T = tile_geom(H, c.n, g.N, g.E, c.B)[0]
    lv = g.N + 1000 if variant == "live_past_n" else None
    live = None if lv is None else torch.tensor([lv, g.B], dtype=torch.int64, device="cuda")
    out, _, acc = c.forward(live)
    tag = f"{variant} H={H}"
    assert torch.equal(out, ref_out), f"out differs from pert_tconv_fwd_c ({tag})"
    _check_stats(c, out, acc, lv, T, tag)


# ------------------------------------------------------------------------------------------------------ c
LIN_N = [4096, 4097, 4159, 51277, 102463]
LIN_LIVE = ["N", "N-1", "64k", "64k-1", "64k+1", "empty_clusters", "1", "past_N"]


def _lin_live(N, kind):
    k = (N // 64) // 2
    return {"N": N, "N-1": N - 1, "64k": 64 * k, "64k-1": 64 * k - 1, "64k+1": 64 * k + 1,
            "empty_clusters": 64 * ((N // 64) // 3) + 17, "1": 1, "past_N": N + 4096}[kind]


@pytest.mark.parametrize("kind", LIN_LIVE)
@pytest.mark.parametrize("N", LIN_N)
def test_linear_bwd_sums(N, kind):
    """pert_linear_bwd_planes_ex: the fp64 column sums of dz and dz xhat over the rows below live[0] (clamped to N),
    added to non-zero contents, at relu_scale 1 and 1 / (1 - 0.1), with exact ReLU zeros in y and shifted / constant
    columns in x; dX bit-identical to pert_linear_bwd_planes, dW4 / db4 within test_gpu_linear_bwd's bars."""
    L = _L()
    H = 64
    assert L.lib().pert_linear_bwd_planes_supported(N, H, H, H) == 1
    nl = _lin_live(N, kind)
    n = min(nl, N)
    gen = torch.Generator(device="cuda").manual_seed(N * 7 + len(kind))
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=gen)   # noqa: E731
    dY = rnd(4, N, H)
    y = torch.relu(rnd(N, H))                                         # exact zeros on about half the entries
    x = rnd(N, H) * 1.5 + 0.3
    x[:, 8:16] += 1e2
    x[:, 16:24] += 1e3
    x[:, CONST_COL] = CONST_VAL
    xd = x[:n].double()
    mean = xd.mean(0).float()
    rstd = (1.0 / torch.sqrt(xd.var(0, unbiased=False) + EPS)).float()
    assert float(rstd[CONST_COL]) == RSTD_CONST
    W4 = rnd(4 * H, H) / math.sqrt(H)
    W4t = W4.t().contiguous()
    live = torch.tensor([nl, 1], dtype=torch.int64, device="cuda")

    def run(dW, db, dX, sums, scale):
        if sums is None:
            L.call("pert_linear_bwd_planes", _ptr(dY), N * H, _ptr(y), H, _ptr(W4t), 4 * H, _ptr(dW), H, _ptr(db),
                   _ptr(dX), H, N, H, H, H, _st())
        else:
            L.call("pert_linear_bwd_planes_ex", _ptr(dY), N * H, _ptr(y), H, _ptr(W4t), 4 * H, _ptr(dW), H, _ptr(db),
                   _ptr(dX), H, N, H, H, H, _ptr(x), _ptr(mean), _ptr(rstd), scale, _ptr(live), _ptr(sums), _st())

    dX_r = torch.full((N * H + 64,), SENT, device="cuda")
    run(torch.zeros(4 * H, H, device="cuda"), torch.zeros(4 * H, device="cuda"), dX_r, None, 1.0)
    Yd = dY.double().permute(1, 0, 2).reshape(N, 4 * H)
    rW, rb = Yd.t() @ y.double(), Yd.sum(0)
    tiles = math.ceil(N / 64)
    Ds = 2 * math.ceil(tiles / 16) + 1
    xh = (x[:n].double() - mean.double()) * rstd.double()
    for scale in (1.0, float(np.float32(1.0 / (1.0 - 0.1)))):
        tag = f"N={N} live={kind}({nl}) scale={scale:.6g}"
        dW0, db0 = rnd(4 * H, H), rnd(4 * H)
        dW, db = dW0.clone(), db0.clone()
        dX = torch.full((N * H + 64,), SENT, device="cuda")
        s0 = torch.randn(2 * H, dtype=torch.float64, device="cuda", generator=gen) * 10
        sums = torch.cat([s0, torch.full((16,), SENT, dtype=torch.float64, device="cuda")])
        run(dW, db, dX, sums, scale)
        torch.cuda.synchronize()
        assert torch.equal(dX, dX_r), f"dX differs from pert_linear_bwd_planes ({tag})"
        assert bool((sums[2 * H:] == SENT).all()), f"memory after the sums written ({tag})"
        for got, want, what, tol in ((dW.double() - dW0.double(), rW, "dW4", 3e-5),
                                     (db.double() - db0.double(), rb, "db4", 2e-5)):
            assert_close(got, want, rtol=tol, what=f"{what} {tag}", norm_only=True)
            assert_close(got, want, rtol=5 * tol, what=f"{what} {tag} (element-wise)")
        dz = (dX[:N * H].view(N, H)[:n] * scale) * (y[:n] > 0)            # fp32, rounded as __fmul_rn
        dz = dz.double()
        a, b = dz.sum(0), (dz * xh).sum(0)
        Ea = Ds * U * dz.abs().sum(0) + 4 * U64 * (s0.abs()[:H] + a.abs())
        Eb = (Ds + 3) * U * (dz * xh).abs().sum(0) + 4 * U64 * (s0.abs()[H:] + b.abs())
        _assert_bar(sums[:H] - s0[:H], a, Ea, f"sum dz ({tag})")
        _assert_bar(sums[H:2 * H] - s0[H:], b, Eb, f"sum dz xhat ({tag})")
        assert float((sums[H + CONST_COL] - s0[H + CONST_COL]).abs()) == 0.0, f"constant column: xhat = 0 ({tag})"


# ------------------------------------------------------------------------------------------------------ d
def _bn_fold_case(g, n_rpc=8, tables=True, hint=True, nl=None, seed=0, name=""):
    """pert_tconv_bwd_bn against fp64 of 'BatchNorm backward at the fp32 mean / rstd, then conv backward'."""
    L, H, N = _L(), 64, g.N
    nl = N if nl is None else nl
    assert L.lib().pert_tconv_bwd_bn_supported(H, n_rpc if tables else 0) == 1
    c = _Conv(g, H, n_rpc, tables, hint, inputs=make_inputs(g, H, n_rpc, tables))
    gen = torch.Generator().manual_seed(seed + N)
    x = torch.randn(N, H, generator=gen) * 1.7 + 0.4
    x[:, 8:12] += 1e3
    x[:, CONST_COL] = CONST_VAL
    xd = x[:nl].double()
    mean = xd.mean(0).float()
    rstd = (1.0 / torch.sqrt(xd.var(0, unbiased=False) + EPS)).float()
    gamma, beta = 1 + 0.3 * torch.randn(H, generator=gen), 0.3 * torch.randn(H, generator=gen)
    scale = float(np.float32(1.0 / 0.9)) if seed % 2 else 1.0
    y = torch.relu((x - mean) * rstd * gamma + beta)
    if scale != 1.0:
        y = y * (torch.rand(N, H, generator=gen) >= 0.1).float() * scale
    dx = torch.randn(N, H, generator=gen)
    dz32 = (dx * scale) * (y > 0)                                   # fp32 products, as bn_bwd_dz4 rounds them
    dz = dz32[:nl].double()
    xh = (x[:nl].double() - mean.double()) * rstd.double()
    a, b = dz.sum(0), (dz * xh).sum(0)
    sums = torch.cat([a, b]).cuda()
    dg0, db0 = torch.randn(H, generator=gen), torch.randn(H, generator=gen)
    dgam = torch.cat([dg0, torch.full((4,), SENT)]).cuda()
    dbet = torch.cat([db0, torch.full((4,), SENT)]).cuda()
    cu = lambda t: t.cuda().contiguous()                            # noqa: E731
    xc, yc, dxc, meanc, rstdc, gammac = map(cu, (x, y, dx, mean, rstd, gamma))
    live = torch.tensor([nl, g.B], dtype=torch.int64, device="cuda") if nl != N else None
    out, alpha, _ = c.forward(stats=False)
    E = g.E
    gbuf = torch.full((N * H + 64,), SENT, device="cuda")
    d = torch.full((3, N * H + 64), SENT, device="cuda")
    dsp = torch.full((E + 64,), SENT, device="cuda")
    rpc_ws = torch.empty(16 * N, device="cuda")
    dt_if = torch.zeros_like(c.t_if) if tables else None
    dt_rpc = torch.zeros_like(c.t_rpc) if tables else None
    bn = L.PertBnBwd(_ptr(dxc), _ptr(yc), _ptr(xc), _ptr(meanc), _ptr(rstdc), _ptr(gammac), _ptr(sums), _ptr(dgam),
                     _ptr(dbet), _ptr(live), scale)
    gi, pl = c.gi, c.pl
    L.call("pert_tconv_bwd_bn", _ptr(gbuf), H, _ptr(pl[0]), _ptr(pl[1]), _ptr(pl[2]), H, _ptr(gi.rowptr),
           _ptr(gi.csr_src), _ptr(c.csr_if), _ptr(c.csr_rpc), _ptr(gi.colptr), _ptr(gi.csc_pos), _ptr(gi.csc_dst),
           _ptr(c.t_if), _ptr(c.t_rpc), _ptr(alpha), _ptr(d[0]), _ptr(d[1]), _ptr(d[2]), H, _ptr(dsp), _ptr(rpc_ws),
           _ptr(dt_if), _ptr(dt_rpc), c.n, N, E, c.B, H, H, ctypes.byref(bn), _st())
    torch.cuda.synchronize()
    tag = f"{name} n_rpc={n_rpc} tables={tables} hint={hint} live={nl} scale={scale:.6g}"
    # g
    ga, rs = gamma.double(), rstd.double()
    g64 = torch.zeros(N, H, dtype=torch.float64)
    g64[:nl] = ga * rs * (dz - a / nl - xh * b / nl)
    gbar = ga.abs() * rs * 10 * U * (dz.abs() + a.abs() / nl + xh.abs() * b.abs() / nl)
    gk = gbuf[:N * H].view(N, H).cpu()
    _assert_bar(gk[:nl], g64[:nl], gbar, f"g ({tag})")
    if nl < N:
        assert bool((gk[nl:] == 0).all()) and not bool(torch.signbit(gk[nl:]).any()), f"ghost rows of g ({tag})"
    assert bool((gbuf[N * H:] == SENT).all()), f"memory after g written ({tag})"
    _assert_bar(dbet[:H].cpu(), db0.double() + a, 2 * U * (db0.double().abs() + a.abs()), f"dbeta += ({tag})")
    _assert_bar(dgam[:H].cpu(), dg0.double() + b, 2 * U * (dg0.double().abs() + b.abs()), f"dgamma += ({tag})")
    assert bool((dgam[H:] == SENT).all()) and bool((dbet[H:] == SENT).all()), f"dgamma / dbeta past H ({tag})"
    # the conv backward at the fp64 g
    q, k, v, s, t_if, t_rpc, _ = c.cpu
    src, dst = torch.from_numpy(g.src), torch.from_numpy(g.dst)
    ia, ib = torch.from_numpy(g.if_id), torch.from_numpy(g.rpc_id(max(n_rpc, 1)))
    want = _ref_run(q, k, v, s, t_if, t_rpc, src, dst, ia, ib, g64)
    bar = _bar_of(name)
    for z, key in enumerate(("dq", "dk", "dv")):
        assert_close(d[z, :N * H].view(N, H).cpu(), want[key], rtol=bar, what=f"{key} ({tag})")
        assert bool((d[z, N * H:] == SENT).all()), f"memory after {key} written ({tag})"
    if tables:
        assert_close(dt_if.cpu(), want["dt_if"], rtol=TABLE_BAR, what=f"dt_if ({tag})")
        assert_close(dt_rpc.cpu(), want["dt_rpc"], rtol=TABLE_BAR, what=f"dt_rpc ({tag})")
    if E:
        # ds = dL/d<q_i, k_j + e> per edge: alpha_t (<g_i, v_j + e_t> - <g_i, out_i - s_i>) / sqrt(H), CSR order
        qd, kd, vd = q.double(), k.double(), v.double()
        vj = vd[src]
        if tables:
            vj = vj + t_if.double()[ia] + t_rpc.double()[ib]
        _, al = ref_tconv(qd, kd, vd, None, src, dst, ia, ib, t_if.double() if tables else None,
                          t_rpc.double() if tables else None)
        gv = (g64[dst] * vj).sum(-1)
        mix = torch.zeros(N, dtype=torch.float64).index_add_(0, dst, al * gv)
        ds = al * (gv - mix[dst]) / math.sqrt(H)
        assert_close(dsp[:E].cpu(), ds[gi.perm.long().cpu()], rtol=bar, what=f"ds ({tag})")
    assert bool((dsp[E:] == SENT).all()), f"memory after ds written ({tag})"


@pytest.mark.parametrize("variant", ["rpc1", "rpc8", "rpc9", "rpc64", "no_tables", "no_hint", "live"])
@pytest.mark.parametrize("name", list(BUILDERS))
def test_conv_bwd_bn(name, variant):
    g = graph(name)
    kw = {"rpc1": dict(n_rpc=1), "rpc8": dict(n_rpc=8), "rpc9": dict(n_rpc=9, seed=1), "rpc64": dict(n_rpc=64),
          "no_tables": dict(tables=False, seed=1), "no_hint": dict(hint=False),
          "live": dict(nl=g.N - g.N // 3 - 1, seed=1)}[variant]
    _bn_fold_case(g, name=name, **kw)


def test_conv_bwd_bn_one_node():
    g = Graph([1], np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0))
    _bn_fold_case(g, name="one_node")


def test_conv_bwd_bn_rejects_65_rpc_types():
    """n_rpc = 65 (a 16.25 KiB rpc table): PERT_ERR_UNSUPPORTED and nothing written."""
    L, H = _L(), 64
    g = graph("dense")
    c = _Conv(g, H, 65, True, inputs=make_inputs(g, H, 65, True))
    N, E = g.N, g.E
    buf = torch.zeros(N * H, device="cuda")
    gbuf = torch.full((N * H,), SENT, device="cuda")
    d = torch.full((3, N * H), SENT, device="cuda")
    sums = torch.zeros(2 * H, dtype=torch.float64, device="cuda")
    p = _ptr(buf)
    bn = L.PertBnBwd(p, p, p, p, p, p, _ptr(sums), p, p, None, 1.0)
    gi, pl = c.gi, c.pl
    rc = L.lib().pert_tconv_bwd_bn(_ptr(gbuf), H, _ptr(pl[0]), _ptr(pl[1]), _ptr(pl[2]), H, _ptr(gi.rowptr),
                                   _ptr(gi.csr_src), _ptr(c.csr_if), _ptr(c.csr_rpc), _ptr(gi.colptr), _ptr(gi.csc_pos),
                                   _ptr(gi.csc_dst), _ptr(c.t_if), _ptr(c.t_rpc), p, _ptr(d[0]), _ptr(d[1]),
                                   _ptr(d[2]), H, p, None, _ptr(torch.zeros_like(c.t_if)),
                                   _ptr(torch.zeros_like(c.t_rpc)), 65, N, E, g.B, H, H, ctypes.byref(bn), _st())
    torch.cuda.synchronize()
    assert rc == UNSUPPORTED
    assert bool((gbuf == SENT).all()) and bool((d == SENT).all())


# ------------------------------------------------------------------------------------------------------ e
SHIFT_COLS = (3, 5, 7)


def _shift(oracle):
    """lin_skip biases of every conv shifted by 1e2 on SHIFT_COLS; conv output column CONST_COL made constant (its
    rows of the value, skip and edge weights and of the value bias zeroed: out = the skip bias there)."""
    with torch.no_grad():
        for conv in oracle.convs:
            conv.lin_skip.bias[list(SHIFT_COLS)] += 1e2
            conv.lin_value.weight[CONST_COL] = 0.0
            conv.lin_value.bias[CONST_COL] = 0.0
            conv.lin_skip.weight[CONST_COL] = 0.0
            conv.lin_edge.weight[CONST_COL] = 0.0


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("H", [32, 48, 64, 128])
def test_engine_step_shifted_activations(H, p):
    """One cfg2 training step against the fp32 / fp64 oracles: gradients and BatchNorm running statistics."""
    from tests.test_gpu_any_width import _parity

    _, b = _parity(2, None, H, p=p, tag=f"shifted cfg2 H={H} p={p}", prep=_shift)
    assert b.x.size(0) >= 4096


@pytest.mark.parametrize("H", [48, 64])
def test_bucketed_step_shifted_activations(H):
    """A padded batch (capacity bucket, live rows below the capacity) on the shifted model: the bucketed step matches
    the eager step, BatchNorm running statistics included."""
    from pert_gnn_kdd23_b200.train import BucketedTrainStep, FlatParams, FusedAdam, fused_train_step
    from tests.helpers import is_structural_zero_grad, make_batch
    from tests.test_gpu_any_width import _models

    d = make_batch(2, 40, seed=5).to("cuda")
    _, ma = _models(2, H, prep=_shift)
    mb = copy.deepcopy(ma)
    oa, ob = FusedAdam(FlatParams(ma), lr=1e-3), FusedAdam(FlatParams(mb), lr=1e-3)
    step = BucketedTrainStep(mb, ob, 0.5)
    for n in range(2):
        la = fused_train_step(ma, oa, d, 0.5)
        lb = step(d)
        assert_close(lb, la, rtol=1e-4, what=f"bucketed H={H} loss step {n}")
    assert step.capture_error is None, step.capture_error
    assert_close(mb._engine.bn_running, ma._engine.bn_running, rtol=1e-4, what=f"H={H} BN running statistics")
    pa = dict(ma.named_parameters())
    for name, prm in mb.named_parameters():
        if is_structural_zero_grad(name, len(ma.convs)):
            continue
        logit = any(t in name for t in (".lin_query.", ".lin_key.", ".lin_edge."))
        assert_close(prm, pa[name], rtol=2e-2 if logit else 2e-3, norm_only=logit, what=f"bucketed H={H} {name}")
