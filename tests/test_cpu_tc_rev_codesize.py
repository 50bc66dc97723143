"""CPU-only: the reverse-mode tensor-core MLP kernel k_mlp_tc<3> (sdf, feature and d sdf / d x_c) keeps its epilogue bodies inside
the instruction-cache budget, read from the library's SASS.

The epilogues are unrolled straight-line code and run at their arithmetic pace only while a body fits the SM's instruction cache
(a 22 KB body does, a 37 KB one never does: DESIGN.md §3.1).  The kernel once had seven bodies of 16-45 KB (16 048 instructions,
251 KB).  Instructions are attributed to the epilogue call site in the kernel that they were inlined from (`nvdisasm -gi` line
info; the library is built with -lineinfo)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL = "_ZN4hold8k_mlp_tcILi3EEEvNS_6TcArgsE"
BODY_LIMIT = 1408            # 22 KB of 16-byte instructions
KERNEL_LIMIT = 8000


def instructions_per_call_site(lib_path, kernel, workdir):
    """{outermost source line of mlp_tc.cuh: SASS instructions inlined from it} over the kernel's text section."""
    if shutil.which("cuobjdump") is None or shutil.which("nvdisasm") is None:
        pytest.skip("cuobjdump / nvdisasm unavailable")
    subprocess.run(["cuobjdump", "-xelf", "all", lib_path], cwd=workdir, check=True, capture_output=True)
    cubins = sorted(f for f in os.listdir(workdir) if f.endswith(".cubin"))
    assert cubins, "no sm_90a cubin in the library"
    counts, inside, line = {}, False, None
    for cubin in cubins:
        out = subprocess.run(["nvdisasm", "-gi", os.path.join(workdir, cubin)], capture_output=True, text=True, check=True).stdout
        for s in out.splitlines():
            if s.startswith("//---------------------"):
                inside = s.split()[1] == ".text." + kernel
                line = None
            elif not inside:
                continue
            elif s.lstrip().startswith("//## File"):
                sites = re.findall(r'"([^"]+)", line (\d+)', s)
                line = int(sites[-1][1]) if sites and os.path.basename(sites[-1][0]) == "mlp_tc.cuh" else None
            elif re.match(r"\s+/\*[0-9a-f]{4,6}\*/\s+\S", s):
                counts[line] = counts.get(line, 0) + 1
        if counts:
            break
    return counts


def test_reverse_mode_epilogues_fit_the_instruction_cache_budget(built, tmp_path):
    from hold_b200 import capi

    counts = instructions_per_call_site(capi.LIB_PATH, KERNEL, str(tmp_path))
    total = sum(counts.values())
    with open(os.path.join(ROOT, "hold_b200", "csrc", "mlp_tc.cuh")) as f:
        src = f.read().splitlines()
    # epilogue bodies: the kernel's call sites of the reverse-mode epilogue functions (rev_*)
    bodies = {n: (src[n - 1].strip(), c) for n, c in counts.items() if n is not None and re.search(r"\brev_\w+\s*[<(]", src[n - 1])}
    for n, (text, c) in sorted(bodies.items(), key=lambda kv: -kv[1][1]):
        print(f"line {n:5d} {c:6d} instructions {16 * c / 1024:6.1f} KB  {text}")
    print(f"k_mlp_tc<3>: {total} SASS instructions ({16 * total / 1024:.0f} KB)")
    assert len(bodies) >= 3, bodies        # forward, feature and backward bodies at least
    assert total < KERNEL_LIMIT, total
    worst = max(c for _, c in bodies.values())
    assert worst <= BODY_LIMIT, bodies
