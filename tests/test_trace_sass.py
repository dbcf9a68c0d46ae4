"""What ptxas made of the wavefront trace kernels' traversal state, shared-memory stack and postponed-leaf list
(gfxexp_b200/csrc/wavefront.cuh, traverse.cuh), read from the built library with cuobjdump.

The stack's first entries and the postponed leaves are dynamically indexed per-thread arrays kept in shared memory, laid out
[entry][thread]; the deeper stack entries live in a local array of their own.  Were any of them part of the traversal state,
the whole state would live in local memory: every node step would reload the ray and its position in the tree from there, and
a pointer to the shared arrays loaded from there is generic, so every push, pop and postponed leaf would compile to a generic
LD / ST.  That leaves every result unchanged, so only the machine code shows it.  No GPU is needed."""
import os
import re
import shutil
import subprocess

import pytest

from gfxexp_b200 import abi

# the persistent-thread tracers: ReSTIR visibility, path-tracer and NRC extension / shadow rays, C-ABI ray batches
WAVEFRONT = re.compile(r"k_traceWavefront")


def _cuobjdump():
    for candidate in (shutil.which("cuobjdump"),
                      os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if candidate and os.path.exists(candidate):
            return candidate
    pytest.skip("cuobjdump not found")


@pytest.fixture(scope="module")
def sass():
    """kernel (mangled name) -> its opcodes, predicates stripped"""
    if not os.path.exists(abi.LIB_PATH):
        pytest.skip("library not built")
    text = subprocess.run([_cuobjdump(), "-sass", abi.LIB_PATH], check=True, capture_output=True, text=True).stdout
    kernels, current = {}, None
    for line in text.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            current = kernels.setdefault(m.group(1), [])
            continue
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if m and current is not None:
            current.append(m.group(1))
    return kernels


def test_wavefront_stack_and_pending_leaves_are_shared_memory(sass):
    names = [k for k in sass if WAVEFRONT.search(k)]
    assert any("k_traceWavefrontDeferred" in k for k in names) and any("k_traceWavefrontILb" in k for k in names), \
        "wavefront trace kernels missing from the library"
    for k in names:
        ops = sass[k]
        generic = sorted({op for op in ops if op.split(".")[0] in ("LD", "ST")})
        assert not generic, f"{k}: generic loads / stores {generic}"
        assert any(op.startswith("STS") for op in ops) and any(op.startswith("LDS") for op in ops), \
            f"{k}: no shared-memory stack"


def test_visibility_tracer_keeps_its_state_in_registers(sass):
    """the postponed-leaf visibility kernels touch local memory only for the stack entries beyond the shared part (one push
    and one pop site); with the state in local memory they had 57 local loads and stores"""
    names = [k for k in sass if "k_traceWavefrontDeferred" in k]
    assert names
    for k in names:
        local = [op for op in sass[k] if op.split(".")[0] in ("LDL", "STL")]
        assert len(local) <= 8, f"{k}: {len(local)} local loads / stores"
