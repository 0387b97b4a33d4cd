"""The ordering rule of programmatic dependent launch (csrc/common.cuh), checked over the text of csrc/*.cu.

A kernel launched through launch_pdl / launch_pdl_cluster may start while its predecessor still runs.  Such a kernel
must call pdl_wait(); it may call pdl_trigger() only after pdl_wait(); and before pdl_wait() its body stores nothing to
global memory.  The check reads kernel bodies only (not the device functions they call), which is where the split
between set-up and work is made."""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pert_gnn_kdd23_b200", "csrc")

_KERNEL = re.compile(r"__global__\s+(?:void\s+)?(?:__launch_bounds__\s*\([^)]*\)\s*)?(\w+)\s*\(")
_FUNC = re.compile(r"(\w+)\s*\(([^()]*)\)\s*\{")
_LAUNCH = re.compile(r"\blaunch_pdl(_cluster)?\s*\(")
# stores to global memory: PTX stores / reductions, the vector helpers, bulk shared -> global copies, atomics on
# anything but shared arrays, and element assignments through the kernel's argument struct (a. / g.)
_GLOBAL_STORE = [
    re.compile(r"st\.global|red\.global|\bred\.|bulk_s2g"),
    re.compile(r"\b(?:st4|red4)\s*\("),
    re.compile(r"\batomic\w*\s*\(\s*(?!&?s_|&?S\.)"),
    re.compile(r"\b[ag]\.[\w.]+\s*\[[^\]]*\]\s*(?:[-+*/|&^]?=)(?!=)"),
]


def strip_comments(src):
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    return re.sub(r"//[^\n]*", "", src)


def _match(src, i, open_ch, close_ch):
    """Index one past the bracket that closes the one at src[i]."""
    depth = 0
    for j in range(i, len(src)):
        if src[j] == open_ch:
            depth += 1
        elif src[j] == close_ch:
            depth -= 1
            if depth == 0:
                return j + 1
    raise ValueError("unbalanced")


def kernels(src):
    """{kernel name: body text} of every __global__ function of a comment-free source."""
    out = {}
    for m in _KERNEL.finditer(src):
        args_end = _match(src, m.end() - 1, "(", ")")
        brace = src.index("{", args_end)
        if ";" in src[args_end:brace]:
            continue                                  # a declaration
        out[m.group(1)] = src[brace:_match(src, brace, "{", "}")]
    return out


def _call_args(src, open_paren):
    """Top-level comma-separated arguments of the call whose '(' is at open_paren."""
    end = _match(src, open_paren, "(", ")")
    args, depth, cur = [], 0, ""
    for ch in src[open_paren + 1:end - 1]:
        if ch in "(<[" :
            depth += 1
        elif ch in ")>]":
            depth -= 1
        if ch == "," and depth == 0:
            args.append(cur.strip())
            cur = ""
        else:
            cur += ch
    args.append(cur.strip())
    return args


def pdl_launched(src):
    """Names of the kernels a source launches through launch_pdl / launch_pdl_cluster, directly or through a function
    that forwards its kernel parameter to them."""
    names = set()
    for m in _LAUNCH.finditer(src):
        args = _call_args(src, m.end() - 1)
        if not args or not args[0]:
            continue                                      # the template definitions themselves
        kern = re.match(r"\w+", args[1] if m.group(1) else args[0])
        if kern is None:
            continue
        kern = kern.group(0)
        if kern == "kernel" and "KArgs" in src[max(0, m.start() - 400):m.start()]:
            continue                                      # launch_pdl forwarding to launch_pdl_cluster
        fwd = [f for f in _FUNC.finditer(src[:m.start()]) if re.search(rf"\b{kern}\b", f.group(2))]
        if fwd:                                           # a forwarder: the kernels are its callers' first arguments
            f = fwd[-1].group(1)
            for c in re.finditer(rf"\b{f}\s*\(", src):
                a = _call_args(src, c.end() - 1)
                k = re.match(r"\w+", a[0]) if a and a[0] else None
                if k and not re.fullmatch(r"\w+\s+\w+", a[0]):   # not the forwarder's own parameter list
                    names.add(k.group(0))
        else:
            names.add(kern)
    return names


def violations(src):
    """Rule violations of one comment-free source, as strings."""
    bodies = kernels(src)
    out = []
    for name in sorted(pdl_launched(src)):
        body = bodies.get(name)
        if body is None:
            out.append(f"{name}: launched through launch_pdl but not defined in the same file")
            continue
        if "pdl_wait()" not in body:
            out.append(f"{name}: launched through launch_pdl without pdl_wait()")
    for name, body in bodies.items():
        w = body.find("pdl_wait()")
        t = body.find("pdl_trigger()")
        if t >= 0 and (w < 0 or t < w):
            out.append(f"{name}: pdl_trigger() before pdl_wait()")
        if w >= 0:
            pre = body[:w]
            for pat in _GLOBAL_STORE:
                hit = pat.search(pre)
                if hit:
                    out.append(f"{name}: global store before pdl_wait(): {hit.group(0)!r}")
    return out


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


@pytest.mark.parametrize("name", sources())
def test_pdl_rule(name):
    with open(os.path.join(CSRC, name)) as f:
        src = strip_comments(f.read())
    assert violations(src) == []


def test_conv_chain_is_pdl_launched():
    found = set()
    for name in sources():
        with open(os.path.join(CSRC, name)) as f:
            found |= pdl_launched(strip_comments(f.read()))
    assert {"k_bn_linear_fwd_planes", "k_tile_fwd", "k_tile_bwd_dst", "k_tile_bwd_src",
            "k_linear_bwd_planes"} <= found, found


_BAD = """
__global__ void __launch_bounds__(256) k_nowait(Args a) { a.out[0] = 1.f; }
__global__ void k_early_trigger(Args a) { pdl_trigger(); pdl_wait(); }
__global__ void k_early_store(Args a) { red4(a.p, v); pdl_wait(); }
__global__ void k_early_atomic(Args a) { atomicAdd(a.p, 1.f); pdl_wait(); }
__global__ void k_early_member(Args g) { g.mean[c] = mu; pdl_wait(); }
__global__ void k_good(Args a) { __shared__ int s_h[4]; atomicAdd(&s_h[0], 1); float x = a.q[0]; pdl_wait();
  pdl_trigger(); a.out[0] = x; }
template <typename K> int fwd(K kernel, int grid, const Args& a, cudaStream_t st) {
  return launch_pdl(kernel, grid, 256, 0, st, a); }
int run(const Args& a, cudaStream_t st) {
  launch_pdl(k_early_trigger, 1, 32, 0, st, a);
  launch_pdl_cluster(4, k_good, 4, 32, 0, st, a);
  return fwd(k_nowait<4, true>, 1, a, st);
}
"""


def test_checker_finds_each_violation():
    src = strip_comments(_BAD)
    assert pdl_launched(src) == {"k_nowait", "k_early_trigger", "k_good"}
    v = violations(src)
    assert any(s.startswith("k_nowait: launched through launch_pdl without") for s in v), v
    assert any(s.startswith("k_early_trigger: pdl_trigger() before") for s in v), v
    for k in ("k_early_store", "k_early_atomic", "k_early_member"):
        assert any(s.startswith(f"{k}: global store before") for s in v), (k, v)
    assert not any(s.startswith("k_good") for s in v), v
