"""What a per-run reduction costs in a warp that holds several runs (lanes of run g: the aligned segment of Wq = 2^lg lanes g * Wq
.. g * Wq + Wq - 1, as in the packed-lanes kernel).  At Wq = 1, 2, 4, 8, 16 (and 32: one run per warp) it times, in a dependent
chain of ITERS reductions per warp at full occupancy (2 CTAs of 1024 threads per SM):
  redux.*  __reduce_{or,add,max}_sync over the run's sub-warp mask (a divergent fallback below Wq = 32: one REDUX per run);
  seg_*    the segmented butterflies of kernel_common.cuh (full-mask shuffles);
  ballot   one flag ORed over the run: a ballot masked to the run's lanes;
  bal.max  the run's highest word with a nonzero bit word and that word's highest bit: ballot, masked, FLO, one shuffle, FLO
           (the floor cut's hs_p in frontier_pack.cu);
  base     the chain's own arithmetic without a collective.
Prints SM cycles per reduction and warp (clock64 over the chain), and the same minus `base`.  The kernel is compiled at run time
(nvcc, sm_90a) into a temporary directory."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bobrapet_b200", "csrc")
NVCC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
ITERS = int(os.environ.get("ITERS", "4096"))

SRC = r"""
#include "kernel_common.cuh"
using namespace bf;

template <int OP>
__global__ void __launch_bounds__(1024, 2) probe(uint32_t lg, uint32_t iters, unsigned long long* cyc, uint32_t* sink) {
  const uint32_t lane = threadIdx.x & 31u, Wq = 1u << lg;
  const uint32_t gmask = (Wq == 32u ? FULL : ((1u << Wq) - 1u)) << ((lane >> lg) << lg);
  uint32_t v = lane * 0x9E3779B9u;
  __syncwarp();
  const long long t0 = clock64();
  for (uint32_t i = 0; i < iters; ++i) {
    const uint32_t x = (v + i + lane) & 0x3FFu;
    if (OP == 0) v = x;
    if (OP == 1) v = __reduce_or_sync(gmask, x);
    if (OP == 2) v = __reduce_add_sync(gmask, x);
    if (OP == 3) v = __reduce_max_sync(gmask, x);
    if (OP == 4) v = seg_or(x, lg);
    if (OP == 5) v = seg_add(x, lg);
    if (OP == 6) v = seg_max(x, lg);
    if (OP == 7) v = (__ballot_sync(FULL, x & 1u) & gmask) != 0u ? x : x + 1u;
    if (OP == 8) {
      const uint32_t tb = __ballot_sync(FULL, x != 0u) & gmask;
      const uint32_t hl = 31u - __clz(tb), hb = __shfl_sync(FULL, x, hl);
      v = tb ? (hl & (Wq - 1u)) * 32u + 32u - __clz(hb) : 0u;
    }
  }
  const long long t1 = clock64();
  if (lane == 0) atomicAdd(cyc, (unsigned long long)(t1 - t0));
  if (v == 0x7FFFFFFFu) sink[0] = v;   // keeps the chain
}

extern "C" int sm_count() {
  int n = 0;
  return cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0) == cudaSuccess ? n : -1;
}

extern "C" int run(int op, uint32_t lg, uint32_t iters, int blocks, unsigned long long* cyc_out, float* ms_out) {
  static void (*const fns[9])(uint32_t, uint32_t, unsigned long long*, uint32_t*) = {
      probe<0>, probe<1>, probe<2>, probe<3>, probe<4>, probe<5>, probe<6>, probe<7>, probe<8>};
  unsigned long long* cyc; uint32_t* sink;
  if (cudaMalloc(&cyc, 8) != cudaSuccess || cudaMalloc(&sink, 4) != cudaSuccess) return -1;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  fns[op]<<<blocks, 1024>>>(lg, iters, cyc, sink);   // warm-up
  cudaMemset(cyc, 0, 8);
  cudaEventRecord(e0);
  fns[op]<<<blocks, 1024>>>(lg, iters, cyc, sink);
  cudaEventRecord(e1);
  if (cudaEventSynchronize(e1) != cudaSuccess) return -2;
  cudaEventElapsedTime(ms_out, e0, e1);
  cudaMemcpy(cyc_out, cyc, 8, cudaMemcpyDeviceToHost);
  cudaFree(cyc); cudaFree(sink); cudaEventDestroy(e0); cudaEventDestroy(e1);
  return cudaGetLastError() == cudaSuccess ? 0 : -3;
}
"""

NAMES = ("base", "redux.or", "redux.add", "redux.max", "seg_or", "seg_add", "seg_max", "ballot", "bal.max")


def build(out):
    src = os.path.join(out, "collective_probe.cu")
    with open(src, "w") as f:
        f.write(SRC)
    lib = os.path.join(out, "collective_probe.so")
    subprocess.run([NVCC, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-shared",
                    "--cudart", "static", "-I", CSRC, src, "-o", lib], check=True)
    return lib


def main():
    with tempfile.TemporaryDirectory() as tmp:
        lib = C.CDLL(build(tmp))
        if "--build-only" in sys.argv:
            print("built", lib)
            return
        gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip().splitlines()[0]
        blocks = 2 * lib.sm_count()
        warps = blocks * 32
        print("collective_probe: %d CTAs x 1024 threads, %d dependent reductions per warp; gpu: %s" % (blocks, ITERS, gpu))
        print("SM cycles per reduction and warp (clock64 over the chain); in brackets: minus `base`")
        print("%-10s" % "Wq" + "".join("%18s" % n for n in NAMES))
        for lg in range(6):
            row, base = [], None
            for op in range(len(NAMES)):
                cyc, ms = C.c_ulonglong(0), C.c_float(0)
                rc = lib.run(op, lg, ITERS, blocks, C.byref(cyc), C.byref(ms))
                if rc != 0:
                    raise SystemExit("run(%s, Wq=%d) failed: %d" % (NAMES[op], 1 << lg, rc))
                c = cyc.value / warps / ITERS
                if op == 0:
                    base = c
                    row.append("%18.1f" % c)
                else:
                    row.append("%10.1f (%5.1f)" % (c, c - base))
            print("%-10d" % (1 << lg) + "".join(row))


if __name__ == "__main__":
    main()
