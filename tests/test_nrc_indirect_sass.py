"""GFX_PT_NRC_INDIRECT is a template switch of the NRC path tracer's kernels: the GFX_PT_NRC instantiations (k_nrcFirstHit and
k_nrcBounce with INDIRECT = false, with and without bump mapping) and the blending k_nrcAccumulate must be the machine code they
were before the switch existed.  The digests are those of the kernels k_nrcFirstHit<BUMP>, k_nrcBounce<BUMP> and k_nrcAccumulate
as nvcc 12.9 built them for sm_90a before the switch; every SASS instruction with its operands, read from the built library
with cuobjdump.  No GPU is needed.  The k_nrcBounce digests are those after two later, deliberate fixes of GFX_PT_NRC's
bounce (DESIGN.md): a training path whose rendering path has ended in the cache no longer adds its NEE, emitter and environment
terms to the rendering radiance, and a training suffix ended by a full record buffer no longer feeds its previous record."""
import hashlib
import os
import re
import shutil
import subprocess

import pytest

from gfxexp_b200 import abi

BEFORE = {
    "_ZN3gfx13k_nrcFirstHitILb0ELb0EE": "33fb6ae57af369f30e6d6b6d3d05ccc41f285d2275ae8680ce57283164b28b4c",
    "_ZN3gfx13k_nrcFirstHitILb1ELb0EE": "af5fac04162efb1bebd5ca0bf488a497a6dccb92237c7c0123b6c69e7a8f197c",
    "_ZN3gfx11k_nrcBounceILb0ELb0EE": "f9725facc445abbe56fc6c900a5ac11d2ddb8eb0412a6b5420dad48913b11b93",
    "_ZN3gfx11k_nrcBounceILb1ELb0EE": "023e512a6697b2152289bd87aaa241d0fc424fee701345f86b6cd1095d6219a3",
    "_ZN3gfx15k_nrcAccumulateILb0EE": "1a7513efbcbcc72a5080eef118147cffb3ce90d485fd31b927d1fe9aa85ff0de",
}


def _tool(name):
    for candidate in (shutil.which(name), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)):
        if candidate and os.path.exists(candidate):
            return candidate
    pytest.skip(f"{name} not found")


def test_nrc_kernels_match_their_recorded_sass():
    if not os.path.exists(abi.LIB_PATH):
        pytest.skip("library not built")
    version = subprocess.run([_tool("nvcc"), "--version"], capture_output=True, text=True).stdout
    if "release 12.9" not in version:
        pytest.skip("the digests are nvcc 12.9's")
    text = subprocess.run([_tool("cuobjdump"), "-sass", abi.LIB_PATH], check=True, capture_output=True, text=True).stdout
    kernels, current = {}, None
    for line in text.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            current = kernels.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?;)", line)
        if m and current is not None:
            current.append(m.group(1))
    for prefix, digest in BEFORE.items():
        names = [k for k in kernels if k.startswith(prefix)]
        assert len(names) == 1, (prefix, names)
        got = hashlib.sha256("\n".join(kernels[names[0]]).encode()).hexdigest()
        assert got == digest, f"{names[0]}: the SASS of the GFX_PT_NRC kernel changed"
    # the switch's own instantiations exist
    assert any(k.startswith("_ZN3gfx13k_nrcFirstHitILb0ELb1EE") for k in kernels)
    assert any(k.startswith("_ZN3gfx15k_nrcAccumulateILb1EE") for k in kernels)
