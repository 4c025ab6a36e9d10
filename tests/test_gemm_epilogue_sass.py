"""CPU: the tensor-core GEMM epilogue issues every global load of a tile before its first store.

C, the residual and act'(pre) operand are plain pointers that may alias (C == residual is allowed), so the compiler keeps
a load written after a store behind it.  An epilogue that loads one row pair and stores it before loading the next waits
for one memory round trip per row pair (2 BN / 8 per thread and tile) while every SM sits idle; loading the whole
fragment first waits for one.  This reads the machine code of every gemm_wgmma_kernel instantiation and checks that,
after the last HGMMA, no LDG follows an STG.  It reads the built libmmx.so, or a cubin compiled from gemm_wgmma.cu with
the build's flags, and skips when neither cuobjdump nor a way to make the code is available."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "transformer-mm-explainability_b200")


def _tool(name):
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    path = os.path.join(cuda, "bin", name)
    return path if os.path.exists(path) else shutil.which(name)


@pytest.fixture(scope="module")
def sass(tmp_path_factory):
    cuobjdump = _tool("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    binary = os.path.join(PKG, "libmmx.so")
    if not os.path.exists(binary):
        nvcc = _tool("nvcc")
        if nvcc is None:
            pytest.skip("neither libmmx.so nor nvcc available")
        import importlib.util
        spec = importlib.util.spec_from_file_location("mmx_build_flags", os.path.join(PKG, "build.py"))
        build = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(build)
        binary = str(tmp_path_factory.mktemp("sass") / "gemm_wgmma.cubin")
        subprocess.run([nvcc, *build.FLAGS, "-cubin", os.path.join(PKG, "csrc", "gemm_wgmma.cu"), "-o", binary],
                       check=True, capture_output=True)
    out = subprocess.run([cuobjdump, "-sass", binary], check=True, capture_output=True, text=True).stdout
    return out


def _functions(text):
    """{mangled name: [opcode, ...]} of the gemm_wgmma_kernel instantiations in a cuobjdump -sass listing."""
    funcs, name = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if "gemm_wgmma_kernel" in m.group(1) else None
            if name:
                funcs[name] = []
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if name and m:
            funcs[name].append(m.group(1))
    return funcs


def test_no_load_after_store_in_epilogue(sass):
    funcs = _functions(sass)
    # 3 modes (3xTF32, fp16x3 in-kernel split, fp16x3 pre-split) x 3 tile widths x with / without act
    assert len(funcs) == 18, sorted(funcs)
    for name, ops in funcs.items():
        last = max(i for i, op in enumerate(ops) if op.startswith("HGMMA"))
        stored, late = False, []
        for op in ops[last + 1:]:
            if op.startswith("STG"):
                stored = True
            elif op.startswith("LDG") and stored:
                late.append(op)
        assert not late, f"{name}: {len(late)} global loads issued after a store in the epilogue"
