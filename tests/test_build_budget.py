"""Register / spill budget of the hot kernels, read from the `-Xptxas -v` output of the in-tree build (no GPU
needed). A change in a shared header (protocol.h is inlined into every fused kernel) that pushes a hot kernel over
its register budget silently costs 30 % of the step time; this test makes that loud."""
import glob
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOGS = os.path.join(ROOT, "build", "adapm_b200")


def kernel_name(name):
    """a kernel's name as the tests use it, e.g. ``transe_step_kernel<3, 1, true>``: demangled (c++filt) if mangled,
    without the project's namespaces, cut at the argument list"""
    if name.startswith("_Z"):
        name = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip()
    name = name.replace("(anonymous namespace)::", "").replace("adapm::cudaops::", "").replace("adapm::", "")
    return re.sub(r"^void ", "", name).split("(")[0]


def _kernels():
    logs = glob.glob(os.path.join(LOGS, "*.cu.o.log"))
    if not logs:
        from adapm_b200 import _build

        _build.build()
        logs = glob.glob(os.path.join(LOGS, "*.cu.o.log"))
    out = {}
    pat = re.compile(r"Compiling entry function '([^']+)' for 'sm_90a'\n(?:ptxas info\s*:\s*Function properties[^\n]*\n"
                     r"\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n)?"
                     r"ptxas info\s*:\s*Used (\d+) registers")
    for f in logs:
        for name, stack, st, ld, regs in pat.findall(open(f).read()):
            out[kernel_name(name)] = {"regs": int(regs), "spill": int(st or 0) + int(ld or 0)}
    return out


def test_hot_kernel_instantiations_stay_within_their_register_budget():
    k = _kernels()
    if not k:
        pytest.skip("no ptxas logs (extension was not built in-tree)")
    # full-register variants of the fused steps: 2 blocks x 256 threads x 128 registers = the register file, no spills
    # (sgns_step_tma_kernel<VPL, MAXREG>)
    for name in ("sgns_step_tma_kernel<3, 128>", "sgns_step_tma_kernel<2, 128>", "sgns_step_tma_kernel<1, 128>",
                 "sgns_step_kernel<3>", "kge_step_kernel<2>", "mf_step_kernel<1>"):
        assert name in k, sorted(k)
        assert k[name]["regs"] <= 128 and k[name]["spill"] == 0, (name, k[name])
    # lean multi-GPU variant: 104 registers leave 12 K registers per SM for one block of the round kernels
    lean = k["sgns_step_tma_kernel<3, 104>"]
    assert lean["regs"] <= 104 and lean["spill"] <= 256, lean
    # the round's kernels must fit NEXT to two lean training blocks: meta passes (128-thread blocks, no spills) and
    # the row pass (128 threads)
    room = 65536 - 2 * 256 * 104
    for name, v in k.items():
        if name.startswith(("phase_meta_kernel", "phase_scan_kernel", "phase_b_")):
            assert v["regs"] * 128 <= room and v["spill"] == 0, (name, v)
    assert k["phase_row_kernel<float>"]["regs"] * 128 <= room, k["phase_row_kernel<float>"]
    # tensor-core kernels: no spills, enough room for 1 CTA/SM with large smem tiles
    for name, v in k.items():
        if name.startswith(("gemm_nt_wgmma", "gather_gemm_kernel")):
            assert v["spill"] == 0, (name, v)


def test_hopper_instructions_are_in_the_built_extension():
    """SASS / PTX of the in-tree extension (cuobjdump, no GPU needed): the kernels that are documented to use the Hopper
    tensor cores (wgmma), TMA, mbarriers and NVLS multimem really contain those instructions - a refactoring that silently drops
    one of them (e.g. a fallback path becoming the only path) fails here, not in a benchmark weeks later."""
    import shutil

    so = glob.glob(os.path.join(ROOT, "adapm_b200", "_C*.so"))
    if not so or shutil.which("cuobjdump") is None:
        pytest.skip("no built extension or no cuobjdump")
    sass = subprocess.run(["cuobjdump", "-sass", so[0]], capture_output=True, text=True).stdout
    per, cur = {}, None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            per[cur] = set()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ln)
        if m and cur:
            per[cur].add(m.group(1).split(".")[0] + ("." + m.group(1).split(".")[1] if m.group(1).startswith(("LDGMC", "UBLK")) else ""))

    def ops_of(fragment):
        hits = [v for k, v in per.items() if fragment in k]
        assert hits, f"no kernel matching {fragment}"
        out = set()
        for h in hits:
            out |= h
        return out

    gemm = ops_of("gemm_nt_wgmma_kernel")
    assert {"HGMMA", "UTMALDG", "SYNCS", "WARPGROUP"} <= gemm, sorted(gemm)   # wgmma bf16, TMA ring, mbarriers
    assert "QGMMA" in gemm                                                       # fp8 (e4m3) instantiation
    gather = ops_of("gather_gemm_kernel")
    assert {"HGMMA", "UTMALDG", "SYNCS"} <= gather, sorted(gather)
    sgns = ops_of("sgns_step_tma_kernel")
    assert {"UBLKCP.S", "UBLKRED.G", "SYNCS"} <= sgns, sorted(sgns)              # TMA ring in, TMA bulk reductions out
    assert {"LDGMC.E"} <= ops_of("xbar_kernel")                                   # multimem.ld_reduce (NVLS)
    ptx = subprocess.run(["cuobjdump", "-ptx", so[0]], capture_output=True, text=True).stdout
    assert "multimem.st.release.sys.global" in ptx and "multimem.ld_reduce" in ptx
    assert "wgmma.mma_async" in ptx and "cp.reduce.async.bulk" in ptx
