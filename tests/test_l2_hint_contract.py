"""The programmatic-dependent-launch rule (csrc/common.cuh) for the L2 forms of the conv chain's stores (csrc/sm90.cuh):
a hinted store and a discard of an L2 line are global writes, so a kernel that waits with pdl_wait() issues neither
before it.  Checked over the kernel bodies of csrc/*.cu with the parser of test_pdl_contract."""
import os
import re

import pytest

from tests.test_pdl_contract import CSRC, kernels, sources, strip_comments

_L2_WRITE = re.compile(r"\b(?:discard_l2|st4_hint|st2_hint)\s*\(|discard\.global")


def l2_violations(src):
    out = []
    for name, body in kernels(src).items():
        w = body.find("pdl_wait()")
        if w >= 0:
            hit = _L2_WRITE.search(body[:w])
            if hit:
                out.append(f"{name}: L2 write before pdl_wait(): {hit.group(0)!r}")
    return out


@pytest.mark.parametrize("name", sources())
def test_no_l2_write_before_pdl_wait(name):
    with open(os.path.join(CSRC, name)) as f:
        assert l2_violations(strip_comments(f.read())) == []


def test_chain_discards_after_the_wait():
    found = {}
    for name in sources():
        with open(os.path.join(CSRC, name)) as f:
            for k, body in kernels(strip_comments(f.read())).items():
                if "discard_l2(" in body:
                    found[k] = body.find("discard_l2(") > body.find("pdl_wait()") >= 0
    assert set(found) == {"k_tile_fwd", "k_tile_bwd_dst", "k_linear_bwd_planes"}, found
    assert all(found.values()), found


def test_checker_finds_early_l2_writes():
    src = strip_comments("""
__global__ void k_early_discard(Args a) { discard_l2(a.p); pdl_wait(); }
__global__ void k_early_hint(Args a) { st4_hint(a.p, v, pol); pdl_wait(); }
__global__ void k_good(Args a) { float4 v = ldg4_hint(a.q, pol); pdl_wait(); st2_hint(a.p, w, pol); discard_l2(a.p); }
""")
    v = l2_violations(src)
    assert any(s.startswith("k_early_discard:") for s in v) and any(s.startswith("k_early_hint:") for s in v), v
    assert not any(s.startswith("k_good") for s in v), v
