"""The k-loops of the wgmma GEMM and convolution kernels carry no memory barrier.

Every stage of `wg_mainloop` is released by an mbarrier arrive (on the peer CTA too, in the
2-CTA kernels).  A `.release.cluster` arrive compiles to MEMBAR.ALL.GPU in front of it, which
stalls the consumer warp until all its earlier stores (the previous tile's epilogue) are
acknowledged, once per k-block.  This reads `cuobjdump -sass` of the in-tree library, as
`tools/sass_summary.py` does, and checks every GEMM and convolution instantiation: no MEMBAR
between the first warpgroup MMA and the last WARPGROUP.DEPBAR.  Needs nvcc and cuobjdump, not
a GPU.
"""
import re
import shutil
import subprocess

import pytest

KERNELS = ("gemm_wgmma_kernel", "conv_wgmma_kernel")


def _sass_by_kernel(lib_path):
    out = subprocess.run(["cuobjdump", "-sass", lib_path], capture_output=True, text=True,
                         check=True).stdout
    kernels, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if any(k in m.group(1) for k in KERNELS) else None
            if name:
                kernels[name] = []
            continue
        if name is None:
            continue
        ins = re.search(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", line)
        if ins:
            kernels[name].append(ins.group(1))
    return kernels


@pytest.mark.skipif(shutil.which("nvcc") is None or shutil.which("cuobjdump") is None,
                    reason="needs nvcc to build the sm_90a library and cuobjdump to read its SASS")
def test_no_membar_inside_wgmma_k_loops():
    from opendwm_b200 import build
    kernels = _sass_by_kernel(build.build())
    for k in KERNELS:
        assert any(k in n for n in kernels), "no %s in the library" % k
    bad = []
    for name, ops in kernels.items():
        # HGMMA: 16-bit operands, QGMMA: E4M3
        first = next(i for i, op in enumerate(ops) if op.startswith(("HGMMA", "QGMMA")))
        last = max(i for i, op in enumerate(ops) if op.startswith("WARPGROUP.DEPBAR"))
        n = sum(op.startswith("MEMBAR") for op in ops[first:last])
        if n:
            bad.append("%s: %d MEMBAR" % (name, n))
    assert not bad, "memory barriers inside the wgmma k-loop:\n" + "\n".join(bad)
