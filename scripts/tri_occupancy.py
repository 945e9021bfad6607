"""Registers, spills, shared memory and resident CTAs per SM of the eight tri_node_kernel<SLAB, VP, FAST> instantiations.

  python scripts/tri_occupancy.py          # compile only (no GPU): ptxas figures and the CTAs/SM they allow on an H100
  python scripts/tri_occupancy.py --gpu    # also build a small harness and ask the driver (cudaOccupancy...)

Shared memory is given at the staging capacity of hypersim100 (N x K = 200 match rows per node, one candidate slot per
row, three with VPs), rounded the way lm_tri_run rounds it. Everything is compiled in a temporary directory."""
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from limap_b200 import _build  # noqa: E402
from limap_b200.synth import CONFIGS  # noqa: E402

SRC = os.path.join(_build.CSRC, "tri_kernels.cu")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
THREADS = 128
# sm_90 (H100): 64K registers and 228 KB of shared memory per SM, 1 KB of it reserved per CTA, at most 16 CTAs of 128
# threads; registers are allocated per warp in units of 256, shared memory in units of 128 bytes
SM_REGS, SM_SMEM, CTA_RESERVED, MAX_CTAS = 65536, 233472, 1024, 16
INSTANTIATIONS = [(s, v, f) for s in (False, True) for v in (False, True) for f in (False, True)]


def name(inst):
    return "<%s>" % ", ".join("true" if b else "false" for b in inst)


def smem_bytes(cap, fast):  # tri_smem_bytes() in tri_kernels.cu
    return cap * (16 * 8 + 4 * 8 + 32 + 8 + 4 + 2 + 4 * 2) if fast else cap * (17 * 8 + 48 + 8) + 4 * 2 * (cap + 96) * 4 + 4 * cap * 2


def hypersim100_cap(vp, fast):
    cfg = CONFIGS["hypersim100"]
    slots = cfg["N"] * cfg["K"] * (3 if vp else 1)
    step = 8 if fast else 32
    return -(-slots // step) * step


def ptxas(extra=()):
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [NVCC] + _build.NVCC_FLAGS + ["-Xptxas", "-v", *extra, "-c", "-o", os.path.join(tmp, "tri.o"), SRC]
        out = subprocess.run(cmd, check=True, capture_output=True, text=True).stderr
    res, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Compiling entry function '_ZN2lm15tri_node_kernelILb(\d)ELb(\d)ELb(\d)E", line)
        if m:
            cur = tuple(bool(int(g)) for g in m.groups())
            res[cur] = {}
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            res[cur]["spill_st"], res[cur]["spill_ld"] = int(m.group(1)), int(m.group(2))
        m = re.search(r"Used (\d+) registers.*?(\d+) bytes smem", line)
        if m:
            res[cur]["regs"], res[cur]["static_smem"] = int(m.group(1)), int(m.group(2))
            cur = None
    return res


def ctas_per_sm(regs, smem):
    per_warp = -(-regs * 32 // 256) * 256
    by_regs = SM_REGS // (per_warp * (THREADS // 32))
    per_cta = -(-(smem + CTA_RESERVED) // 128) * 128
    by_smem = SM_SMEM // per_cta
    return min(by_regs, by_smem, MAX_CTAS), by_regs, by_smem


HARNESS = r"""
#include "tri_kernels.cu"
template <bool SLAB, bool VP, bool FAST> static void query(size_t smem) {
  auto k = lm::tri_node_kernel<SLAB, VP, FAST>;
  if (SLAB) smem = 0;
  if (smem > 48 * 1024) cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (!SLAB && !VP && FAST) // as launch_tri_vf sets it
    cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
  int n = -1;
  const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k, lm::kThreads, smem);
  printf("<%s, %s, %s> dynamic smem %zu B: %d CTAs/SM%s%s\n", SLAB ? "true" : "false", VP ? "true" : "false",
         FAST ? "true" : "false", smem, n, e == cudaSuccess ? "" : " error: ", e == cudaSuccess ? "" : cudaGetErrorString(e));
}
int main(int argc, char **argv) {
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("%s, %d SMs, %zu B shared memory per SM\n", prop.name, prop.multiProcessorCount, prop.sharedMemPerMultiprocessor);
  query<false, false, false>(atol(argv[1])); query<false, false, true>(atol(argv[2]));
  query<false, true, false>(atol(argv[3])); query<false, true, true>(atol(argv[4]));
  query<true, false, false>(0); query<true, false, true>(0); query<true, true, false>(0); query<true, true, true>(0);
  return 0;
}
"""


def gpu_occupancy():
    with tempfile.TemporaryDirectory() as tmp:
        src, exe = os.path.join(tmp, "occ.cu"), os.path.join(tmp, "occ")
        with open(src, "w") as f:
            f.write(HARNESS)
        subprocess.run([NVCC] + _build.ARCH + ["-O3", "-std=c++17", "-I", _build.CSRC, "-o", exe, src], check=True)
        args = [str(smem_bytes(hypersim100_cap(vp, fast), fast)) for vp in (False, True) for fast in (False, True)]
        print(subprocess.run([exe] + args, check=True, capture_output=True, text=True).stdout, end="")


def main():
    res = ptxas()
    print("tri_node_kernel<SLAB, VP, FAST>, 128 threads, compiled for sm_90a; shared memory at the hypersim100 cap")
    print("%-22s %5s %9s %9s %5s %12s %11s" % ("instantiation", "regs", "spill st", "spill ld", "cap", "dyn smem", "CTAs/SM"))
    for inst in INSTANTIATIONS:
        slab, vp, fast = inst
        r = res[inst]
        cap = hypersim100_cap(vp, fast)
        dyn = 0 if slab else smem_bytes(cap, fast)
        n, by_regs, by_smem = ctas_per_sm(r["regs"], dyn + r["static_smem"])
        print("%-22s %5d %7d B %7d B %5d %10d B %4d (regs %d, smem %d)"
              % (name(inst), r["regs"], r["spill_st"], r["spill_ld"], cap, dyn, n, by_regs, by_smem))
    if "--gpu" in sys.argv:
        gpu_occupancy()


if __name__ == "__main__":
    main()
