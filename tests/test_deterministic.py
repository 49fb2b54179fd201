"""Deterministic mode, host side: argument checks and workspace sizes of the atomic-free entry points, the training
dispatch following torch.use_deterministic_algorithms, and (compiled for sm_90a, no GPU needed) the absence of floating-point
atomics from the deterministic kernels."""
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "raft-ncup_b200", "csrc")
P = 4096                                                  # any non-null, 16-byte aligned address: nothing is dereferenced


@pytest.fixture
def det():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=False)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def test_wgrad_det_workspace_and_argument_checks():
    from rnc import native
    L = native.lib()
    ws = L.rnc_conv2d_cl_wgrad_workspace_bytes
    # 3x3 64->64 at half resolution: 24576 pixels, 352 blocks wanted per tap -> 80 pixels per block, 308 splits
    assert ws(64, 64, 2, 96, 128, 3, 3, 1) == 308 * (9 * 64 * 64 + 64) * 4
    # whatever the layer, the partials stay within one 64x64 tile for each of the 132 * 24 blocks
    for shape in ((64, 64, 8, 220, 512, 3, 3, 1), (324, 256, 8, 55, 128, 1, 1, 1), (256, 126, 8, 55, 128, 3, 3, 1),
                  (4, 64, 8, 440, 1024, 7, 7, 2), (384, 128, 8, 55, 128, 1, 5, 1)):
        assert ws(*shape) <= 132 * 24 * (64 * 64 + 64) * 4, shape
    # a small layer keeps its split: B*H*W = 2*14*19 = 532 pixels in blocks of 64 -> 9 splits
    assert ws(128, 256, 2, 14, 19, 3, 3, 1) == 9 * (9 * 128 * 256 + 256) * 4
    assert ws(64, 64, 2, 96, 128, 3, 3, 2) <= ws(64, 64, 2, 96, 128, 3, 3, 1)
    for bad in ((0, 64, 2, 8, 8, 3, 3, 1), (6, 64, 2, 8, 8, 3, 3, 1), (64, 64, 2, 8, 8, 2, 3, 1), (64, 64, 2, 8, 8, 3, 3, 3),
                (64, 64, 0, 8, 8, 3, 3, 1), (64, 64, 2, 8, 8, 9, 9, 1)):
        assert ws(*bad) == 0, bad
    f = L.rnc_conv2d_cl_wgrad_det
    nb = ws(64, 32, 2, 8, 8, 3, 3, 1)

    def call(cin=64, ldx=64, ldg=32, ldw=32, x=P, gw=P, w=P, wsb=nb):
        return f(x, ldx, cin, P, ldg, 32, 2, 8, 8, 3, 3, 1, gw, ldw, P, w, wsb, None)

    assert call(cin=6, ldx=8) == -1 and call(ldx=62) == -1 and call(ldg=16) == -1 and call(ldw=16) == -1
    assert call(x=None) == -2 and call(gw=None) == -2 and call(w=None) == -2 and call(x=P + 4) == -2 and call(ldg=34) == -2
    assert call(wsb=nb - 4) == -5


def test_lookup_det_workspace_and_argument_checks():
    from rnc import native
    L = native.lib()
    ws = L.rnc_corr_lookup_bwd_workspace_bytes
    B, H, W = 2, 48, 64
    n = 4 * B * H * W
    cells = sum(B * ((H >> l) + 9) * ((W >> l) + 9) for l in range(4))
    up = lambda v: (v + 255) // 256 * 256                     # noqa: E731
    # staging [levels][pixels][100] floats, two key and two row buffers, cell starts, the sort's scratch
    assert ws(B, H, W, 4) == up(n * 400) + 4 * up(n * 4) + up((cells + 1) * 4) + up((1 << 20) + n * 4)
    assert ws(B, H, W, 2) < ws(B, H, W, 4)
    assert ws(0, H, W, 4) == 0 and ws(B, H, W, 5) == 0 and ws(B, 4, W, 4) == 0
    f = L.rnc_corr_lookup_bwd_det
    nb = ws(B, H, W, 4)

    def call(B=B, D=256, levels=4, radius=4, ldg=324, f1=P, g2=P, w=P, wsb=nb):
        return f(f1, P, P, P, ldg, B, D, H, W, levels, radius, P, g2, w, wsb, None)

    assert call(B=0) == -1 and call(levels=0) == -1 and call(levels=5) == -1
    assert call(D=128) == -3 and call(radius=3) == -3 and call(ldg=323) == -3
    assert call(f1=None) == -2 and call(g2=None) == -2 and call(w=None) == -2 and call(w=P + 8) == -2
    assert call(wsb=nb - 1) == -5


def test_instnorm_det_workspace_and_argument_checks():
    from rnc import native
    L = native.lib()
    ws = L.rnc_instnorm_stats_det_workspace_bytes
    assert ws(4, 3072, 64) == 4 * 6 * 64 * 16 and ws(4, 3073, 64) == 4 * 7 * 64 * 16
    assert ws(0, 64, 64) == 0 and ws(4, 64, 130) == 0 and ws(4, 64, 66) == 0
    f = L.rnc_instnorm_stats_det
    nb = ws(2, 1000, 64)

    def call(N=2, C=64, x=P, w=P, mr=P, wsb=nb):
        return f(x, N, 1000, C, 1e-5, w, wsb, mr, None)

    assert call(N=0) == -1 and call(C=132) == -1 and call(C=62) == -1
    assert call(x=None) == -2 and call(w=None) == -2 and call(mr=None) == -2 and call(w=P + 8) == -2
    assert call(wsb=nb - 8) == -5


class _Recorder:
    """Stands in for librnc: records which entry points a dispatch calls, launches nothing."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append(name)
            return 4096 if name.endswith("_workspace_bytes") else 0
        return fn


@pytest.mark.parametrize("on", [False, True])
def test_training_dispatch_follows_the_flag_at_the_binding(on, monkeypatch, request):
    import rnc.train as tr
    from rnc import native
    if on:
        request.getfixturevalue("det")
    rec = _Recorder()
    monkeypatch.setattr(native, "_lib", rec)
    monkeypatch.setattr(native, "stream", lambda: None)
    assert tr.deterministic() == on
    gw, gb = tr._wgrad(torch.zeros(1, 4, 4, 8), torch.zeros(1, 4, 4, 16), 16, 3, 3, 1, True)
    assert gw.shape == (9, 8, 16) and gb.shape == (16,)
    tr._lookup_bwd(torch.zeros(1, 8, 8, 256), torch.zeros(100), torch.zeros(1, 2, 8, 8), torch.zeros(1, 8, 8, 324), 4)
    want = ["rnc_conv2d_cl_wgrad_workspace_bytes", "rnc_conv2d_cl_wgrad_det"]          # one weight gradient, both modes
    want += ["rnc_corr_lookup_bwd_workspace_bytes", "rnc_corr_lookup_bwd_det"] if on else ["rnc_corr_lookup_bwd"]
    assert rec.calls == want


def _float_atomics(tmp_path, src):
    from rnc.build import ARCH, NVCC_FLAGS, nvcc_path
    obj = tmp_path / (src + ".o")
    cmd = [nvcc_path(), *ARCH, *NVCC_FLAGS, "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-c", os.path.join(CSRC, src),
           "-o", str(obj)]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc_path()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    found, fn = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            found[fn] = []
            continue
        m = re.search(r"\b((?:RED|ATOM)G?\.\S*F(?:16|32|64)\S*)", line)
        if m and fn is not None:
            found[fn].append(m.group(1))
    return found


@pytest.mark.parametrize("src,kernels", [
    ("train_ops.cu", ["conv_wgrad_kernel", "wgrad_reduce_kernel", "corr_lookup_bwd_kernelILb1E", "cell_start_kernel",
                      "lookup_gather_kernel", "DeviceRadixSort"]),
    ("encoder_ops.cu", ["instnorm_stats_kernelILb1E", "instnorm_reduce_kernel"]),
])
def test_deterministic_kernels_have_no_float_atomics(tmp_path, src, kernels):
    try:
        from rnc.build import nvcc_path
        nvcc_path()
    except RuntimeError:
        pytest.skip("nvcc not available")
    found = _float_atomics(tmp_path, src)
    for k in kernels:
        hits = {fn: ops for fn, ops in found.items() if k in fn}
        assert hits, (k, sorted(found))
        assert not any(hits.values()), hits
    # the default lookup backward and InstanceNorm statistics keep their atomics (and the scan finds them)
    atomic = "corr_lookup_bwd_kernelILb0E" if src == "train_ops.cu" else "instnorm_stats_kernelILb0E"
    assert any(ops for fn, ops in found.items() if atomic in fn)
