"""The dense node-linear GEMMs (`pert_gemm_nt`, `pert_gemm_tn`, `pert_colsum`: csrc/gemm.cu, csrc/gemm_tc.cu) against
float64, at every kernel variant and every dispatch boundary.

Each entry point picks its kernel from the shape at run time. `expected_kernel` restates that choice; a CPU test checks
that CASES reach every variant, and a GPU test runs every case inside one `torch.profiler` session and compares the
kernels each launched with the restatement.

Reference and bar: ref = A64 . B64^T (+ bias) in float64 on the device, and for every element

    |C - ref|_ij <= tau * (|A| . |B|^T + |bias|)_ij            (+ |C0|_ij when the call adds into C0)

so rows and columns whose terms cancel are held to the size of their terms, not to the tensor's rms. The taus follow
DESIGN section 3's error model (u = 2^-24, the unit roundoff of fp32):

  * exact-fp32 SIMT kernels: recursive summation with fma, tau = (K + 3) u (K terms, bias, one += into C0);
  * 3xTF32 wgmma kernels (a = hi + lo, hi the nearest tf32): the product error is lo_a.hi_b and hi_a.lo_b with lo cut to
    tf32 by the tensor core (2^-21 |a||b| each) plus the dropped lo_a.lo_b (2^-22), within 3 * 2^-21; the tensor-core
    accumulator truncates, at most one fp32 ulp (2 u) of the running sum per wgmma, three wgmmas per K-step of 8:
        NT  tau = 3 * 2^-21 + 3 ceil(Kp / 8) * 2u + (P + 1) u     (Kp = K of one plane, P planes added with red.global)
        TN  tau = 3 * 2^-21 + 12 * 2u + (ceil(R / 32) + 2) u      (32-row tensor-core sums, added with round to nearest)

DESIGN's norm-wise bars (max |C - ref| / max |ref|) are checked as well where DESIGN promises them: tensor-core NT
2e-6 (K <= 144) up to 8e-6 (K = 512), tensor-core TN 3e-5, on ordinary operands. The stress cases (columns and rows
scaled by 1e4 and 1e-4, terms of 1e3 that cancel exactly) have results far smaller than their terms, and only the
element-wise bar speaks to them.

Memory a call does not own (C's padding columns, rows past M, the columns of each plane a blocked C leaves out, a guard
after C) is filled with a sentinel and must be unchanged afterwards; A's padding holds NaN, which would poison any
output that read it. Every measured error goes to $PERT_PARITY_LOG when it is set.
"""
import json
import math
import os
import re
import subprocess
import sys
import tempfile
import zlib
from dataclasses import dataclass

import pytest
import torch

from tests.helpers import RTOL, assert_close, assert_grads_close

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
SENTINEL = 12345.0
GUARD = 256                     # floats after C, and rows past M in every plane of C
SMEM_MAX = 226 * 1024           # csrc/gemm_tc.cu
NT_BN = (16, 32, 48, 64, 80, 96, 112, 128)
TN_NCP = tuple(range(16, 161, 16))


# ------------------------------------------------------------------------------------------------------------ bars
def tau_simt(K):
    return (K + 3) * U


def tau_tc_nt(Kp, planes=1):
    return 3 * 2.0 ** -21 + 3 * math.ceil(Kp / 8) * 2 * U + (planes + 1) * U


def tau_tc_tn(R):
    return 3 * 2.0 ** -21 + 12 * 2 * U + (math.ceil(R / 32) + 2) * U


def norm_bar_nt(K):
    """DESIGN section 3: 2e-6 up to K = 144, 8e-6 at K = 512 (linear in between); no promise beyond K = 512."""
    if K <= 144:
        return 2e-6
    return 2e-6 + 6e-6 * (K - 144) / (512 - 144) if K <= 512 else None


NORM_BAR_TN = 3e-5


def bar_ratio(got, ref, mag, tau):
    """max_ij |got - ref| / (tau * mag): <= 1 passes the element-wise bar (an element with mag = 0 must be exact)."""
    err = (got.double() - ref).abs()
    lim = tau * mag
    if bool((err[lim == 0] != 0).any()):
        return math.inf
    return float((err / lim.clamp_min(1e-300)).max()) if err.numel() else 0.0


def _log(**kw):
    path = os.environ.get("PERT_PARITY_LOG")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(kw) + "\n")


def check_bar(got, ref, mag, tau, what, norm_bar=None):
    r = bar_ratio(got, ref, mag, tau)
    en = float((got.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30)) if ref.numel() else 0.0
    with torch.no_grad():
        eff = float(((got.double() - ref).abs() / mag.clamp_min(1e-300)).max()) if ref.numel() else 0.0
    _log(what=what, tau_bar=tau, tau_measured=eff, norm=en, norm_bar=norm_bar)
    assert r <= 1.0, f"{what}: element-wise error {r:.3g} x the bar (tau {tau:.3e}, measured {eff:.3e}, norm {en:.3e})"
    if norm_bar is not None:
        assert en <= norm_bar, f"{what}: norm-wise error {en:.3e} > {norm_bar:.1e}"


# ------------------------------------------------------------------------------------------------------------ dispatch
@dataclass(frozen=True)
class Nt:
    M: int
    Nc: int
    K: int
    a_cb: int = 0           # > 0: A stored as K / a_cb planes [M, lda] (plane-blocked, the layout of dq|dk|dv|ds)
    lda: int = 0            # 0: a_cb or K
    c_cb: int = 0           # > 0: C stored as Nc / c_cb planes [M, ldc]
    ldc: int = 0            # 0: c_cb or Nc
    bias: bool = True
    relu: bool = False
    accumulate: bool = False
    stress: bool = False

    def __str__(self):
        s = f"nt-M{self.M}-N{self.Nc}-K{self.K}"
        for k in ("a_cb", "lda", "c_cb", "ldc"):
            if getattr(self, k):
                s += f"-{k}{getattr(self, k)}"
        return s + "".join(f"-{k}" for k in ("relu", "accumulate", "stress") if getattr(self, k)) + \
            ("" if self.bias else "-nobias")


@dataclass(frozen=True)
class Tn:
    R: int
    Mc: int
    Nc: int
    a_cb: int = 0           # > 0: A stored as Mc / a_cb planes [R, a_cb]
    ldb: int = 0
    b_cb: int = 0           # > 0: B stored as Nc / b_cb planes [R, b_cb]
    ldc: int = 0
    colsum: bool = True
    stress: bool = False

    def __str__(self):
        s = f"tn-R{self.R}-M{self.Mc}-N{self.Nc}"
        for k in ("a_cb", "ldb", "b_cb", "ldc"):
            if getattr(self, k):
                s += f"-{k}{getattr(self, k)}"
        return s + ("" if self.colsum else "-nocolsum") + ("-stress" if self.stress else "")


@dataclass(frozen=True)
class Colsum:
    R: int
    Cc: int
    a_cb: int = 0

    def __str__(self):
        return f"colsum-R{self.R}-C{self.Cc}" + (f"-a_cb{self.a_cb}" if self.a_cb else "")


def _nt_layout_ok(M, Nc, K, a_cb, a_cbs, a_pz, c_cb, c_cbs, lda, ldc, a_align, c_align):
    if a_cb <= 0 or a_cb >= K:
        a_cb, a_cbs = K, 0
    if c_cb <= 0:
        c_cb, c_cbs = Nc, 0
    if (K % 8 or K > 1024 or Nc % 16 or lda % 4 or ldc % 2 or c_cb % 16 or a_cbs % 4 or a_pz % 4 or c_cbs % 2
            or a_align % 16 or c_align % 8 or M > 2 ** 31 - 1):
        return False
    return a_cb == K or a_cb % 16 == 0


def _nt_bn(Nc, K):
    """N block of k_gemm_nt_wg: Nc split into equal multiples of 16, at most 128, whose [BN, K] hi + lo block fits."""
    Kp = (K + 7) // 8 * 8
    nblk = (Nc + 127) // 128
    while True:
        if nblk > Nc // 16:
            return None
        if Nc % nblk == 0 and (Nc // nblk) % 16 == 0 and (Nc // nblk) * Kp * 8 <= SMEM_MAX:
            return Nc // nblk
        nblk += 1


def expected_kernel(op, M, Nc, K, a_cb=0, c_cb=0, lda=0, ldc=0, relu=False, accumulate=False, colsum=False, *,
                    a_cbs=0, c_cbs=0, b_cb=0, a_align=16, c_align=16, tc=True):
    """The launches `pert_gemm_nt` (op "nt": C[M,Nc] = A[M,K] . B^T), `pert_gemm_tn` (op "tn": M = R rows, K = Mc output
    rows, ldc of C, `colsum` = a_colsum given) or `pert_colsum` (op "colsum": M = R, Nc = Cc) makes, in order:
    "nt_wg<BN>", "nt_wg<BN>/planes<P>" (after a "memset" of C), "nt_simt", "tn_wg<NCP>", "tn_simt" (after a "colsum"
    when `colsum`) or "colsum". `tc` = False is the PERT_GEMM_TC=0 build of the same call. a_cbs / c_cbs: plane strides
    of blocked A / C; b_cb: a blocked B (tn)."""
    if op == "colsum":
        return ("colsum",)
    if op == "tn":
        R, Mc = M, K
        if a_cb <= 0:
            a_cb, a_cbs = Mc, 0
        if (tc and R >= 4096 and not (0 < b_cb < Nc) and not (Nc % 4 or Nc > 160 or Mc % 2 or a_cb % 2 or lda % 2
                                                               or a_cbs % 2 or ldc % 2 or a_align % 8 or c_align % 8)):
            return (f"tn_wg<{(Nc + 15) // 16 * 16}>",)
        return ("colsum", "tn_simt") if colsum else ("tn_simt",)
    assert op == "nt"
    if a_cb <= 0:
        a_cb = K
    if c_cb <= 0:
        c_cb = Nc
    if tc and M >= 1024 and not accumulate:
        if (a_cb < K and K % a_cb == 0 and not relu and Nc <= 128 and Nc * K * 8 > SMEM_MAX
                and Nc * a_cb * 8 <= SMEM_MAX and K // a_cb <= 8 and c_cb >= Nc
                and _nt_layout_ok(M, Nc, a_cb, a_cb, 0, a_cbs, c_cb, c_cbs, lda, ldc, a_align, c_align)):
            return ("memset", f"nt_wg<{_nt_bn(Nc, a_cb)}>/planes<{K // a_cb}>")
        if _nt_layout_ok(M, Nc, K, a_cb, a_cbs, 0, c_cb, c_cbs, lda, ldc, a_align, c_align):
            bn = _nt_bn(Nc, K)
            if bn is not None:
                return (f"nt_wg<{bn}>",)
    return ("nt_simt",)


# ------------------------------------------------------------------------------------------------------------ cases
def _nt_cases():
    c = []
    for M in (1023, 1024, 1025, 4096 + 63):                                  # the M >= 1024 tensor-core boundary
        c.append(Nt(M, 64, 80))
    for Nc in (16, 32, 48, 64, 80, 96, 112, 128, 144, 176, 256, 33, 120):    # every BN; 144 -> 48, 176 -> 16
        c.append(Nt(2085, Nc, 64))
    c.append(Nt(1100, 1024, 272))                                            # narrowed to BN = 64 by shared memory
    for K in (8, 16, 24, 72, 136, 144, 256, 512, 768, 1024, 1032, 73):      # trailing K-step, K near 1024, fall-backs
        c.append(Nt(4096 + 63, 64, K))
    for K in (144, 256, 512, 768, 1024):                                     # the long-sum accuracy sweep at Nc = 128
        c.append(Nt(4096, 128, K, stress=K in (144, 1024)))
    c += [Nt(2085, 96, 64, bias=False), Nt(2085, 96, 64, relu=True), Nt(2085, 128, 136, bias=False, relu=True),
          Nt(2085, 64, 80, lda=84), Nt(2085, 64, 80, ldc=66), Nt(2085, 64, 80, ldc=65),
          Nt(2085, 256, 80, c_cb=64, ldc=64), Nt(2085, 192, 80, c_cb=64, ldc=68),     # C blocks != the BN = 96 blocks
          Nt(2085, 80, 64, c_cb=20, ldc=20),                                            # c_cb % 16 != 0: falls back
          Nt(2085, 64, 64, a_cb=16), Nt(2085, 64, 192, a_cb=96, lda=100), Nt(2085, 32, 256, a_cb=128),
          Nt(4096, 144, 512, a_cb=128, bias=False),                          # conv-0 dX at H = 128: BN = 48, K = 512
          Nt(2085, 64, 80, accumulate=True), Nt(2085, 18, 40, c_cb=6, ldc=6, accumulate=True),
          Nt(1500, 64, 144, stress=True), Nt(700, 64, 144, stress=True)]
    # deep K over plane-blocked A: gridDim.z planes into a cleared C
    for H, Nc in ((128, 64), (128, 96), (128, 128), (96, 96)):
        c.append(Nt(4096 + 17, Nc, 4 * H, a_cb=H, bias=False))
    c += [Nt(4096 + 17, 128, 512, a_cb=128), Nt(4096 + 17, 128, 512, a_cb=128, ldc=136, bias=False),
          Nt(4096 + 17, 96, 512, a_cb=128, stress=True)]
    # layouts the planes cannot take (Nc % 16 != 0): the exact SIMT kernel
    c += [Nt(4096 + 17, 100, 512, a_cb=128, bias=False), Nt(4096 + 17, 120, 512, a_cb=128, bias=False),
          Nt(4096 + 17, 120, 256, a_cb=64, bias=False), Nt(4096 + 17, 100, 512, a_cb=128, ldc=104)]
    return c


def _tn_cases():
    c = []
    for R in (4095, 4096, 4096 + 31, 51200 + 77):
        c.append(Tn(R, 256, 64))
    for Nc in (4, 16, 20, 32, 48, 64, 80, 96, 112, 128, 144, 152, 160, 164, 9):
        c.append(Tn(8192 + 5, 130, Nc))
    for Mc in (2, 6, 130, 256, 512):
        c.append(Tn(8192 + 5, Mc, 80))
    c += [Tn(8192 + 5, 256, 80, a_cb=64), Tn(8192 + 5, 256, 80, a_cb=64, colsum=False), Tn(8192 + 5, 130, 80,
                                                                                              colsum=False),
          Tn(8192 + 5, 512, 144, a_cb=128), Tn(8192 + 5, 130, 72, ldb=76), Tn(8192 + 5, 128, 64, ldc=66),
          Tn(8192 + 5, 256, 64, b_cb=32), Tn(2000, 256, 80, a_cb=64),
          Tn(51200 + 77, 256, 80, a_cb=64, stress=True), Tn(3000, 130, 64, stress=True)]
    return c


def _colsum_cases():
    c = []
    for R in (1, 63, 64, 10 ** 5):
        for Cc in (1, 33, 512):
            c.append(Colsum(R, Cc))
            if Cc > 1:
                c.append(Colsum(R, Cc, a_cb=11 if Cc == 33 else 128))
    return c


CASES = _nt_cases() + _tn_cases() + _colsum_cases()


def _planes_of(cb, n):
    return n // cb if cb and cb < n else 1


def _nt_geom(c):
    """(lda, a_cbs, planes of A, ldc, c_cbs, planes of C) as the case lays them out."""
    pa = _planes_of(c.a_cb, c.K)
    lda = c.lda or (c.a_cb if pa > 1 else c.K)
    a_cbs = c.M * lda if pa > 1 else 0
    pc = _planes_of(c.c_cb, c.Nc)
    ldc = c.ldc or (c.c_cb if pc > 1 else c.Nc)
    c_cbs = (c.M + GUARD) * ldc if pc > 1 else 0
    return lda, a_cbs, pa, ldc, c_cbs, pc


def _tn_geom(c):
    pa = _planes_of(c.a_cb, c.Mc)
    lda = c.a_cb if pa > 1 else c.Mc
    a_cbs = c.R * lda if pa > 1 else 0
    pb = _planes_of(c.b_cb, c.Nc)
    ldb = c.ldb or (c.b_cb if pb > 1 else c.Nc)
    b_cbs = c.R * ldb if pb > 1 else 0
    return lda, a_cbs, pa, ldb, b_cbs, pb, c.ldc or c.Nc


def expected(c, tc=True):
    if isinstance(c, Colsum):
        return expected_kernel("colsum", c.R, c.Cc, 0)
    if isinstance(c, Tn):
        lda, a_cbs, _, _, _, _, ldc = _tn_geom(c)
        return expected_kernel("tn", c.R, c.Nc, c.Mc, a_cb=c.a_cb, lda=lda, ldc=ldc, colsum=c.colsum, a_cbs=a_cbs,
                               b_cb=c.b_cb, tc=tc)
    lda, a_cbs, pa, ldc, c_cbs, pc = _nt_geom(c)
    return expected_kernel("nt", c.M, c.Nc, c.K, a_cb=c.a_cb if pa > 1 else 0, c_cb=c.c_cb if pc > 1 else 0, lda=lda,
                           ldc=ldc, relu=c.relu, accumulate=c.accumulate, a_cbs=a_cbs, c_cbs=c_cbs, tc=tc)


# ------------------------------------------------------------------------------------------------------------ CPU tests
def test_cases_reach_every_variant():
    seen = {k for c in CASES for k in expected(c)}
    want = {f"nt_wg<{bn}>" for bn in NT_BN} | {f"tn_wg<{n}>" for n in TN_NCP} | {"nt_simt", "tn_simt", "colsum",
                                                                                   "memset"}
    assert want <= seen, sorted(want - seen)
    assert any("/planes<" in k for k in seen)
    # one case behind each guard of the tensor-core path: M < 1024, Nc % 16, K > 1024, K % 8, odd ldc, c_cb % 16,
    # accumulate, the deep-K layouts the planes cannot take, R < 4096, Nc % 4, Nc > 160, blocked B
    for c in (Nt(1023, 64, 80), Nt(2085, 33, 64), Nt(4159, 64, 1032), Nt(4159, 64, 73), Nt(2085, 64, 80, ldc=65),
              Nt(2085, 80, 64, c_cb=20, ldc=20), Nt(2085, 64, 80, accumulate=True),
              Nt(4113, 100, 512, a_cb=128, bias=False), Nt(4113, 120, 256, a_cb=64, bias=False),
              Tn(4095, 256, 64), Tn(8197, 130, 9), Tn(8197, 130, 164), Tn(8197, 256, 64, b_cb=32)):
        assert c in CASES, c
        assert expected(c)[-1] in ("nt_simt", "tn_simt"), (c, expected(c))


def test_restated_dispatch_known_shapes():
    """Spot values of the restatement, worked out by hand from csrc/gemm_tc.cu."""
    assert expected(Nt(2085, 144, 64)) == ("nt_wg<48>",)
    assert expected(Nt(2085, 176, 64)) == ("nt_wg<16>",)
    assert expected(Nt(1100, 1024, 272)) == ("nt_wg<64>",)
    assert expected(Nt(4159, 64, 1024)) == ("nt_wg<16>",)
    assert expected(Nt(4159, 64, 512)) == ("nt_wg<32>",)
    assert expected(Nt(4113, 128, 512, a_cb=128, bias=False)) == ("memset", "nt_wg<128>/planes<4>")
    assert expected(Nt(4113, 96, 384, a_cb=96, bias=False)) == ("memset", "nt_wg<96>/planes<4>")
    assert expected(Nt(4096, 144, 512, a_cb=128, bias=False)) == ("nt_wg<48>",)
    assert expected(Nt(4113, 100, 512, a_cb=128, bias=False)) == ("nt_simt",)
    assert expected(Nt(4159, 64, 80), tc=False) == ("nt_simt",)
    assert expected(Tn(8197, 130, 20)) == ("tn_wg<32>",)
    assert expected(Tn(4095, 256, 64)) == ("colsum", "tn_simt")
    assert expected(Tn(8197, 256, 64, b_cb=32)) == ("colsum", "tn_simt")
    assert expected(Tn(8197, 130, 80, colsum=False), tc=False) == ("tn_simt",)


def _tf32_round(x):
    """Nearest tf32 with the bit trick of tf32_hi (csrc/sm90.cuh): (bits + 0x1000) & 0xffffe000."""
    b = x.float().contiguous().view(torch.int32).to(torch.int64)
    b = ((b + 0x1000) & 0xffffe000) & 0xffffffff
    b = torch.where(b >= 2 ** 31, b - 2 ** 32, b).to(torch.int32)
    return b.view(torch.float32)


def _control_operands(M, Nc, K, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(Nc, K, generator=g) / math.sqrt(K)
    bias = torch.randn(Nc, generator=g)
    A64, B64, b64 = A.double(), B.double(), bias.double()
    ref = A64 @ B64.t() + b64
    mag = A64.abs() @ B64.abs().t() + b64.abs()
    return A, B, bias, ref, mag


@pytest.mark.parametrize("K", [144, 512])
def test_bar_rejects_defects(K):
    """Negative controls: each defect a tensor-core kernel could have must fail the 3xTF32 bar that the exact product
    (rounded once to fp32) passes."""
    M, Nc = 512, 64
    A, B, bias, ref, mag = _control_operands(M, Nc, K, seed=K)
    tau = tau_tc_nt(K)
    assert bar_ratio((A.double() @ B.double().t() + bias.double()).float(), ref, mag, tau) <= 1.0
    # single-pass TF32: operands rounded to tf32, products and sums exact
    tf32 = _tf32_round(A).double() @ _tf32_round(B).double().t() + bias.double()
    assert bar_ratio(tf32, ref, mag, tau) > 1.0
    # one K-step of 8 columns dropped
    keep = torch.ones(K, dtype=torch.float64)
    keep[16:24] = 0
    assert bar_ratio((A.double() * keep) @ B.double().t() + bias.double(), ref, mag, tau) > 1.0
    # two columns of a 16-column chunk swapped in the weights only (a wrong nt_logical_k)
    Bs = B.double().clone()
    Bs[:, [33, 38]] = Bs[:, [38, 33]]
    assert bar_ratio(A.double() @ Bs.t() + bias.double(), ref, mag, tau) > 1.0
    # the deep-K plane path adding the bias once per plane instead of from plane 0 only
    planes = 4
    per_plane_bias = A.double() @ B.double().t() + planes * bias.double()
    assert bar_ratio(per_plane_bias, ref, mag, tau_tc_nt(K // planes, planes)) > 1.0


def test_bar_holds_small_rows_to_their_own_terms():
    """A row far below the tensor's rms (its inputs scaled by 1e-3, as after a cancellation upstream): an error of 1e-3
    of that row's own terms passes the rms-floored element-wise check of tests/helpers, not the tau |A||B| bar."""
    from tests.helpers import elem_err

    M, Nc, K = 256, 64, 144
    A, B, bias, _, _ = _control_operands(M, Nc, K, seed=1)
    A64, B64 = A.double(), B.double()
    A64[6] *= 1e-3
    ref = A64 @ B64.t()
    mag = A64.abs() @ B64.abs().t()
    bad = ref.clone()
    bad[6] += 1e-3 * mag[6]
    assert elem_err(bad, ref) < RTOL
    assert bar_ratio(bad, ref, mag, tau_tc_nt(K)) > 1.0


# ------------------------------------------------------------------------------------------------------------ GPU runs
def _kernel_label(name, grid):
    m = re.search(r"k_gemm_nt_wg<(\d+)>", name)
    if m:
        z = grid[2] if grid and len(grid) > 2 else 1
        return f"nt_wg<{m.group(1)}>" + (f"/planes<{z}>" if z > 1 else "")
    m = re.search(r"k_gemm_tn_wg<(\d+)>", name)
    if m:
        return f"tn_wg<{m.group(1)}>"
    for pat, label in ((r"k_gemm_nt\b(?!_)", "nt_simt"), (r"k_gemm_tn\b(?!_)", "tn_simt"), (r"k_colsum", "colsum")):
        if re.search(pat, name):
            return label
    return None


def launched_per_case(cases, tc=True):
    """Runs the call of every case once inside ONE torch.profiler session (CUDA activity) and returns, per case, the
    GEMM kernels and memsets it launched, in order, labelled as expected_kernel labels them (the plane count is the
    grid's z). Each call sits between two launches of k_relu_bwd, a library kernel no GEMM launches, with the device
    synchronised around them, so the trace cuts into cases even though the inputs are built between the calls."""
    from torch.profiler import ProfilerActivity, profile

    from pert_gnn_kdd23_b200 import _lib

    y, dy = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")

    def cut():
        torch.cuda.synchronize()
        _lib.call("pert_relu_bwd", y.data_ptr(), dy.data_ptr(), 1, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in cases:
            call, _ = setup_case(c, tc)
            cut()
            call()
            cut()
            del call
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    out, cur = [], None
    for e in sorted((e for e in events if e.get("ph") == "X"), key=lambda e: e.get("ts", 0)):
        cat, name = e.get("cat", ""), e.get("name", "")
        if cat == "kernel" and "k_relu_bwd" in name:
            if cur is None:
                cur = []
            else:
                out.append(tuple(cur))
                cur = None
        elif cur is None:
            continue
        elif cat == "gpu_memset" or (cat == "kernel" and name.startswith("Memset")):
            cur.append("memset")
        elif cat == "kernel":
            lab = _kernel_label(name, e.get("args", {}).get("grid"))
            if lab:
                cur.append(lab)
    assert len(out) == len(cases), f"the trace holds {len(out)} complete cases of {len(cases)}"
    return out


def _layout(X, ld, planes):
    """Logical [rows, planes * cols] -> planes x [rows, ld] storage, NaN in the padding columns."""
    rows, n = X.shape
    cols = n // planes
    st = torch.full((planes, rows, ld), float("nan"), device=X.device)
    st[:, :, :cols] = X.view(rows, planes, cols).permute(1, 0, 2)
    return st


def _c_storage(rows, ld, cols, planes):
    """Flat sentinel-filled storage of `planes` x [rows + GUARD, ld] (+ a GUARD tail) and the index of the owned
    [rows, planes * cols] elements."""
    cbs = (rows + GUARD) * ld
    st = torch.full((planes * cbs + GUARD,), SENTINEL, device="cuda")
    p = torch.arange(planes, device="cuda").view(1, planes, 1)
    r = torch.arange(rows, device="cuda").view(rows, 1, 1)
    j = torch.arange(cols, device="cuda").view(1, 1, cols)
    idx = (p * cbs + r * ld + j).reshape(rows, planes * cols)
    return st, idx


def _untouched(st, idx, what):
    mask = torch.ones(st.numel(), dtype=torch.bool, device="cuda")
    mask[idx.reshape(-1)] = False
    assert bool((st[mask] == SENTINEL).all()), f"{what}: memory outside the output was written"


def _stress_nt(A, B, gen):
    M, K = A.shape
    A[:, 1] *= 1e4
    A[:, 2] *= 1e-4
    A[5] *= 1e4
    A[6] *= 1e-4
    r = torch.randn(M, device="cuda", generator=gen)
    j = K - 1                                     # an exactly cancelling pair: column 3 and the last column
    A[:, 3], A[:, j] = 1e3 * r, -1e3 * r
    B[:, j] = B[:, 3]


def setup_nt(c, tc=True):
    from pert_gnn_kdd23_b200 import _lib

    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(str(c).encode()))
    lda, a_cbs, pa, ldc, c_cbs, pc = _nt_geom(c)
    A = torch.randn(c.M, c.K, device="cuda", generator=gen)
    B = torch.randn(c.Nc, c.K, device="cuda", generator=gen) / math.sqrt(c.K)
    if c.stress:
        _stress_nt(A, B, gen)
    Ast = _layout(A, lda, pa)
    bias = torch.randn(c.Nc, device="cuda", generator=gen) if c.bias else None
    ccols = c.Nc // pc
    Cst, idx = _c_storage(c.M, ldc, ccols, pc)
    C0 = torch.randn(c.M, c.Nc, device="cuda", generator=gen) if c.accumulate else None
    if C0 is not None:
        Cst[idx] = C0
    want = expected(c, tc)

    def call():
        _lib.call("pert_gemm_nt", Ast.data_ptr(), lda, c.a_cb if pa > 1 else 0, a_cbs, B.data_ptr(), c.K,
                  bias.data_ptr() if bias is not None else None, Cst.data_ptr(), ldc, c.c_cb if pc > 1 else 0, c_cbs,
                  c.M, c.Nc, c.K, int(c.relu), int(c.accumulate), torch.cuda.current_stream().cuda_stream)

    def check():
        _check_nt(c, A, B, bias, C0, Cst, idx, want)

    return call, check


def _check_nt(c, A, B, bias, C0, Cst, idx, want):
    A64, B64 = A.double(), B.double()
    ref = A64 @ B64.t()
    mag = A64.abs() @ B64.abs().t()
    if bias is not None:
        ref += bias.double()
        mag += bias.double().abs()
    if c.relu:
        ref = ref.clamp_min(0)
    if C0 is not None:
        ref += C0.double()
        mag += C0.double().abs()
    kern = want[-1]
    if kern.startswith("nt_wg"):
        planes = int(kern.split("planes<")[1][:-1]) if "planes" in kern else 1
        tau, nb = tau_tc_nt(c.K // planes, planes), None if c.stress else norm_bar_nt(c.K)
    else:
        tau, nb = tau_simt(c.K), None
    check_bar(Cst[idx], ref, mag, tau, f"{c} {kern}", nb)
    _untouched(Cst, idx, str(c))


def _stress_tn(A, B, gen):
    R = A.shape[0]
    A[:, 1] *= 1e4
    A[:, 0] *= 1e-4
    B[:, 2] *= 1e4
    B[:, 1] *= 1e-4
    A[7] *= 1e4
    A[:64] *= 1e3                                 # rows that cancel exactly against the rows from R / 2
    A[R // 2:R // 2 + 64] = A[:64]
    B[R // 2:R // 2 + 64] = -B[:64]


def setup_tn(c, tc=True):
    from pert_gnn_kdd23_b200 import _lib

    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(str(c).encode()))
    lda, a_cbs, pa, ldb, b_cbs, pb, ldc = _tn_geom(c)
    A = torch.randn(c.R, c.Mc, device="cuda", generator=gen)
    B = torch.randn(c.R, c.Nc, device="cuda", generator=gen)
    if c.stress:
        _stress_tn(A, B, gen)
    Ast, Bst = _layout(A, lda, pa), _layout(B, ldb, pb)
    Cst, idx = _c_storage(c.Mc, ldc, c.Nc, 1)
    C0 = torch.randn(c.Mc, c.Nc, device="cuda", generator=gen)
    Cst[idx] = C0
    cs_st = torch.full((c.Mc + GUARD,), SENTINEL, device="cuda") if c.colsum else None
    cs0 = torch.randn(c.Mc, device="cuda", generator=gen)
    if c.colsum:
        cs_st[:c.Mc] = cs0
    want = expected(c, tc)

    def call():
        _lib.call("pert_gemm_tn", Ast.data_ptr(), lda, c.a_cb if pa > 1 else 0, a_cbs, Bst.data_ptr(), ldb,
                  c.b_cb if pb > 1 else 0, b_cbs, Cst.data_ptr(), ldc, cs_st.data_ptr() if c.colsum else None, c.R,
                  c.Mc, c.Nc, torch.cuda.current_stream().cuda_stream)

    def check():
        _check_tn(c, A, B, C0, cs0, Cst, idx, cs_st, want)

    return call, check


def _check_tn(c, A, B, C0, cs0, Cst, idx, cs_st, want):
    A64, B64 = A.double(), B.double()
    ref = C0.double() + A64.t() @ B64
    mag = C0.double().abs() + A64.abs().t() @ B64.abs()
    kern = want[-1]
    tc_run = kern.startswith("tn_wg")
    check_bar(Cst[idx], ref, mag, tau_tc_tn(c.R) if tc_run else tau_simt(c.R), f"{c} {kern}",
              NORM_BAR_TN if tc_run and not c.stress else None)
    _untouched(Cst, idx, str(c))
    if c.colsum:
        check_bar(cs_st[:c.Mc], cs0.double() + A64.sum(0), cs0.double().abs() + A64.abs().sum(0), tau_simt(c.R),
                  f"{c} {kern} colsum")
        assert bool((cs_st[c.Mc:] == SENTINEL).all()), f"{c}: colsum guard written"


def setup_colsum(c, tc=True):
    from pert_gnn_kdd23_b200 import _lib

    gen = torch.Generator(device="cuda").manual_seed(zlib.crc32(str(c).encode()))
    pa = _planes_of(c.a_cb, c.Cc)
    cols = c.Cc // pa
    A = torch.randn(c.R, c.Cc, device="cuda", generator=gen)
    Ast = _layout(A, cols + 3, pa)
    out = torch.full((c.Cc + GUARD,), SENTINEL, device="cuda")
    o0 = torch.randn(c.Cc, device="cuda", generator=gen)
    out[:c.Cc] = o0

    def call():
        _lib.call("pert_colsum", Ast.data_ptr(), cols + 3, c.a_cb if pa > 1 else 0, c.R * (cols + 3), out.data_ptr(),
                  c.R, c.Cc, torch.cuda.current_stream().cuda_stream)

    def check():
        A64 = A.double()
        check_bar(out[:c.Cc], o0.double() + A64.sum(0), o0.double().abs() + A64.abs().sum(0), tau_simt(c.R), str(c))
        assert bool((out[c.Cc:] == SENTINEL).all()), f"{c}: guard written"

    return call, check


def setup_case(c, tc=True):
    """Inputs of case c on the device -> (call, check): call() launches the GEMM (the kernel expected(c, tc) names),
    check() compares its output with float64 and checks the memory it does not own."""
    return {Nt: setup_nt, Tn: setup_tn, Colsum: setup_colsum}[type(c)](c, tc)


def run_case(c, tc=True):
    call, check = setup_case(c, tc)
    call()
    check()


@gpu
@pytest.mark.parametrize("case", CASES, ids=str)
def test_gemm_vs_fp64(case):
    run_case(case)


def _assert_dispatch(cases, tc=True):
    got = launched_per_case(cases, tc)
    bad = [f"{c}: launched {g}, restated {expected(c, tc)}" for c, g in zip(cases, got) if g != expected(c, tc)]
    assert not bad, "\n".join(bad)


@gpu
def test_gemm_dispatch_matches_restatement():
    """Every case launches exactly the kernels expected_kernel names (and so the variant its bar assumes)."""
    _assert_dispatch(CASES)


def _tc_variant_cases():
    """One case per tensor-core variant (and the plane path), preferring blocked A / C and M >= 1024."""
    pick = {}
    for c in sorted(CASES, key=lambda c: -(bool(getattr(c, "a_cb", 0)) + bool(getattr(c, "c_cb", 0)))):
        k = expected(c)[-1]
        if k.startswith(("nt_wg", "tn_wg")) and k not in pick:
            pick[k] = c
    return list(pick.values())


def test_forced_simt_cases_cover_every_tc_variant():
    kinds = {expected(c)[-1] for c in _tc_variant_cases()}
    assert {f"nt_wg<{bn}>" for bn in NT_BN} | {f"tn_wg<{n}>" for n in TN_NCP} <= kinds
    assert any("/planes<" in k for k in kinds)
    for c in _tc_variant_cases():
        assert expected(c, tc=False)[-1] in ("nt_simt", "tn_simt")


_FORCED = r"""
import sys
sys.path.insert(0, {root!r})
from tests import test_gpu_gemm as t
for c in t._tc_variant_cases():
    t.run_case(c, tc=False)
t._assert_dispatch(t._tc_variant_cases(), tc=False)
print("forced SIMT:", len(t._tc_variant_cases()), "cases")
"""


@gpu
def test_gemm_tc_off_runs_simt_at_tensor_core_shapes():
    """PERT_GEMM_TC=0 (read once per process, so in a child): every tensor-core shape runs on the SIMT kernels and
    passes the SIMT bar."""
    env = dict(os.environ, PERT_GEMM_TC="0")
    p = subprocess.run([sys.executable, "-c", _FORCED.format(root=ROOT)], env=env, cwd=ROOT, capture_output=True,
                       text=True)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]


# ---------------------------------------------------------------------------------------------------------- end to end
@gpu
@pytest.mark.parametrize("Din,H", [(100, 128), (120, 64)])
def test_dropin_conv_whose_data_gradient_leaves_the_plane_path(Din, H):
    """nn.TransformerConv(Din, H).forward(x, edge_index, edge_attr) on 2,048 nodes: the data gradient
    dX = [dq|dk|dv|ds] . W4 has K = 4H and Nc = Din, a deep K whose Nc % 16 != 0 the plane path cannot take. Forward and
    every gradient against the oracle conv in float64."""
    from oracle.model_oracle import OracleTransformerConv
    from pert_gnn_kdd23_b200.nn import TransformerConv

    N, E, De = 2048, 16384, 8
    gen = torch.Generator(device="cuda").manual_seed(Din + H)
    ei = torch.randint(0, N, (2, E), device="cuda", generator=gen)
    torch.manual_seed(0)
    oc = OracleTransformerConv(Din, H, edge_dim=De).double().cuda()
    cc = TransformerConv(Din, H, edge_dim=De)
    cc.load_state_dict({k: v.float() for k, v in oc.state_dict().items()})
    cc = cc.cuda()
    x = torch.randn(N, Din, device="cuda", generator=gen)
    ea = torch.randn(E, De, device="cuda", generator=gen)
    gout = torch.randn(N, H, device="cuda", generator=gen)
    xc = x.clone().requires_grad_()
    yc = cc(xc, ei, ea)
    yc.backward(gout)
    xo = x.double().requires_grad_()
    yo = oc(xo, ei, ea.double())
    yo.backward(gout.double())
    assert_close(yc, yo, rtol=RTOL, what=f"drop-in conv({Din}, {H}) out")
    assert_close(xc.grad, xo.grad, rtol=RTOL, what=f"drop-in conv({Din}, {H}) dx")
    assert_grads_close(cc.named_parameters(), oc.named_parameters(), RTOL)
