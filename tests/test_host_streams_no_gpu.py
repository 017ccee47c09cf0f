"""The host runtime does device work on streams it owns, checks every launch and allocates device memory in one place: no call on the
legacy default stream (which a non-blocking stream does not wait for) or device-wide wait, every kernel launch inside LAUNCH(...), and
cudaMalloc only in DevBuf, DevArena and the prefilter's growable table (PfTable::reserve copies its old contents when it grows)."""
import pathlib
import re

SRC = pathlib.Path(__file__).resolve().parents[1] / "sage_b200" / "csrc" / "sage_b200.cu"
ALLOCATORS = ("struct DevBuf", "struct DevArena", "struct PfTable")


def _lines():
    return SRC.read_text().splitlines()


def test_no_legacy_stream_calls():
    for i, line in enumerate(_lines(), 1):
        for call in ("cudaMemcpy(", "cudaMemset(", "cudaMemcpyToSymbol(", "cudaDeviceSynchronize"):
            assert call not in line, f"sage_b200.cu:{i}: {call} {line.strip()}"


def test_every_launch_is_checked():
    for i, line in enumerate(_lines(), 1):
        if "<<<" in line and not line.lstrip().startswith("#define"):
            assert "LAUNCH(" in line, f"sage_b200.cu:{i}: unchecked launch {line.strip()}"


def test_cuda_malloc_only_in_the_allocators():
    owner = None   # the top-level struct the current line belongs to
    for i, line in enumerate(_lines(), 1):
        if re.match(r"(struct|static|extern|template|class)\b", line):
            owner = next((a for a in ALLOCATORS if line.startswith(a)), None)
        if "cudaMalloc(" in line and "\"" not in line.split("cudaMalloc(")[0]:
            assert owner is not None, f"sage_b200.cu:{i}: cudaMalloc outside {ALLOCATORS}: {line.strip()}"
