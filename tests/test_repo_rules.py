"""CPU: structural rules of this repo that the parity claims rest on — the product never routes through the oracle or
a compiler / CPU fallback, and every GPU test is marked as such."""
import re
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
PKG = ROOT / "panfusion_b200"


def _py(path):
    return [p for p in path.rglob("*.py") if "__pycache__" not in p.parts]


def test_product_never_imports_the_oracle():
    bad = [str(p.relative_to(ROOT)) for p in _py(PKG) if re.search(r"^\s*(from|import)\s+oracle\b", p.read_text(), re.M)]
    assert not bad, f"oracle is test infrastructure only: {bad}"


def test_no_compiler_or_alternative_backends_in_the_product():
    pat = re.compile(r"^\s*(import triton|from triton|import tilelang|from tilelang)|torch\.compile\(|@torch\.compile", re.M)
    bad = [str(p.relative_to(ROOT)) for p in _py(PKG) if pat.search(p.read_text())]
    assert not bad, bad


def test_bench_uses_the_oracle_only_as_the_cpu_baseline():
    src = (ROOT / "bench.py").read_text()
    # the oracle is imported lazily inside the CPU-baseline helpers, never at module level or in run_b200
    head, _, rest = src.partition("def run_b200")
    body_b200 = rest.split("\ndef ", 1)[0]
    assert "oracle" not in body_b200.replace("oracle port", "").replace("_oracle", "")
    assert not re.search(r"^(from|import)\s+oracle\b", src, re.M)


def test_gpu_tests_are_marked():
    for p in (ROOT / "tests").glob("test_gpu_*.py"):
        assert re.search(r"^pytestmark\s*=\s*pytest\.mark\.gpu", p.read_text(), re.M), p.name
    for p in (ROOT / "tests").glob("test_*.py"):
        if not p.name.startswith("test_gpu_") and p.name != Path(__file__).name:
            assert "cuda_device" not in p.read_text(), f"{p.name} uses a GPU fixture but is not a test_gpu_ file"


def test_environment_variables_read_by_the_library():
    """Every layer has one code path: the library reads no environment switch besides these (split-K on/off for the
    bit-identical sharded check, the multi-GPU transport and its forced fallback, the library path, the compiler)."""
    allowed = {"PF_SPLIT_K", "PF_DEVICE_GATHER", "PF_FORCE_IPC_FAIL", "PF_LIB_PATH", "NVCC"}
    read, opaque = set(), []
    for p in PKG.rglob("*"):
        if p.suffix not in (".py", ".cu", ".cuh", ".h") or "__pycache__" in p.parts:
            continue
        for m in re.finditer(r"\b(environ|getenv)\b(.{0,40})", p.read_text()):
            name = re.match(r"""\s*(?:\.get\s*\(|\[|\()\s*["'](\w+)["']""", m.group(2))
            if name:
                read.add(name.group(1))
            else:
                opaque.append(f"{p.relative_to(ROOT)}: {m.group(0)}")
    assert not opaque, f"environment read without a literal name: {opaque}"
    assert read == allowed, f"unexpected: {sorted(read - allowed)}, not found: {sorted(allowed - read)}"
