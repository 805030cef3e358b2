#!/usr/bin/env python
"""Issue rate of bf16 wgmma m64nNk16 on the H100, in the two operand forms the policy forward
(csrc/wdb_mlp.cu) can use: SS (A and B read from shared memory through descriptors) and RS
(A from registers, B from shared memory).

    python scripts/bench_wgmma_forms.py [--iters 4096] [--json OUT]

Builds a small stand-alone CUDA program with nvcc (sm_90a) in a temporary directory and runs
it.  Every CTA (one per SM) has one or two warpgroups; each warpgroup issues `iters` groups of
8 back-to-back MMAs into one of two accumulator sets (one for N = 128; wait_group 1 between groups, as the
forward's slice pipeline does).  Per N in {16, 32, 48, 64, 128}, form and warpgroup count it
reports the SM clocks per MMA (clock64 of CTA 0, so one SM's view), the tensor-core share
(the dense rate of 2048 bf16 FMA per clock per SM, i.e. N / 2 clocks per m64nNk16, over the
measured clocks) and TFLOP/s over all SMs from CUDA events.  The card's name and power limit
are read in the same run.  Prints one JSON object.
"""
import argparse
import json
import os
import subprocess
import tempfile

NS = (16, 32, 48, 64, 128)
GROUP = 8        # MMAs per commit group


def mma_fn(n, rs):
    """Device function issuing one m64n{n}k16 with scale-d = 1 (accumulate)."""
    nr = n // 2
    d = ", ".join(f"%{i}" for i in range(nr))
    outs = ", ".join(f'"+f"(d[{i}])' for i in range(nr))
    if rs:
        a = "{" + ", ".join(f"%{nr + i}" for i in range(4)) + "}"
        b = f"%{nr + 4}"
        ins = '"r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)'
        tail = "1, 1, 1, 0"
    else:
        a, b = f"%{nr}", f"%{nr + 1}"
        ins = '"l"(adesc), "l"(bdesc)'
        tail = "1, 1, 1, 0, 0"
    return f"""
__device__ __forceinline__ void mma_n{n}_{'rs' if rs else 'ss'}(float (&d)[{nr}], const uint32_t *a,
                                                     uint64_t adesc, uint64_t bdesc) {{
  asm volatile("wgmma.mma_async.sync.aligned.m64n{n}k16.f32.bf16.bf16 {{{d}}}, {a}, {b}, {tail};"
               : {outs} : {ins} : "memory");
}}"""


KERNEL = r"""
template <int N, bool RS>
__global__ void __launch_bounds__(256, 1) bench(int iters, long long *clk, float *sink) {
  extern __shared__ __align__(128) unsigned char sm[];
  for (int i = threadIdx.x; i < 16384 / 4; i += blockDim.x) reinterpret_cast<uint32_t *>(sm)[i] = 0x3c003c00u;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const uint32_t base = (uint32_t)__cvta_generic_to_shared(sm);
  const uint64_t adesc = desc(base, 256), bdesc = desc(base + 4096, 256);
  uint32_t a[4] = {0x3c003c00u, 0x3c003c00u, 0x3c003c00u, 0x3c003c00u};
  constexpr int S = N >= 128 ? 1 : 2;   // (two n128 sets do not fit the register file)
  float d[S][N / 2];
#pragma unroll
  for (int s = 0; s < S; s++)
#pragma unroll
    for (int i = 0; i < N / 2; i++) d[s][i] = 0.0f;
  const long long t0 = clock64();
  for (int it = 0; it < iters; it += 2) {
#pragma unroll
    for (int s = 0; s < 2; s++) {
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
      for (int k = 0; k < GROUP; k++) MMA<N, RS>::run(d[s % S], a, adesc, bdesc);
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
    }
  }
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
  __syncthreads();
  const long long t1 = clock64();
  if (blockIdx.x == 0 && threadIdx.x == 0) *clk = t1 - t0;
  float acc = 0.0f;
#pragma unroll
  for (int i = 0; i < N / 2; i++) acc += d[0][i] + d[S - 1][i];
  if (acc == 1234.5f) sink[threadIdx.x] = acc;       // keeps the MMAs alive
}
"""

HOST = r"""
template <int N, bool RS>
void run(int wgs, int iters, int sms) {
  long long *clk; float *sink;
  cudaMalloc(&clk, 8); cudaMalloc(&sink, 4096);
  cudaFuncSetAttribute(bench<N, RS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384);
  for (int w = 0; w < 3; w++) bench<N, RS><<<sms, 128 * wgs, 16384>>>(iters, clk, sink);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e30f; long long c = 0, best_clk = 0;
  for (int r = 0; r < 5; r++) {
    cudaEventRecord(e0);
    bench<N, RS><<<sms, 128 * wgs, 16384>>>(iters, clk, sink);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    cudaMemcpy(&c, clk, 8, cudaMemcpyDeviceToHost);
    if (ms < best) { best = ms; best_clk = c; }
  }
  const cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) { printf("{\"error\": \"%s\"}\n", cudaGetErrorString(err)); exit(1); }
  const double mmas_per_sm = (double)wgs * iters * GROUP;
  const double flop = 2.0 * 64 * N * 16 * mmas_per_sm * sms;
  printf("{\"n\": %d, \"form\": \"%s\", \"warpgroups\": %d, \"clk_per_mma\": %.3f, "
         "\"ideal_clk_per_mma\": %d, \"ms\": %.4f, \"tflops\": %.1f}\n",
         N, RS ? "RS" : "SS", wgs, (double)best_clk / mmas_per_sm, N / 2, best, flop / best / 1e9);
  cudaFree(clk); cudaFree(sink);
}
int main(int argc, char **argv) {
  const int iters = atoi(argv[1]);
  int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (int wgs = 1; wgs <= 2; wgs++) {
RUNS
  }
  return 0;
}
"""


def source():
    parts = ["#include <cstdio>\n#include <cstdlib>\n#include <cstdint>\n",
             f"constexpr int GROUP = {GROUP};",
             """__device__ __forceinline__ uint64_t desc(uint32_t saddr, uint32_t sbo) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)(128 >> 4) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3FFF) << 32);
}
template <int N, bool RS> struct MMA;"""]
    for n in NS:
        for rs in (False, True):
            parts.append(mma_fn(n, rs))
            parts.append(f"""template <> struct MMA<{n}, {'true' if rs else 'false'}> {{
  static __device__ __forceinline__ void run(float (&d)[{n // 2}], const uint32_t *a, uint64_t ad,
                                             uint64_t bd) {{ mma_n{n}_{'rs' if rs else 'ss'}(d, a, ad, bd); }}
}};""")
    parts.append(KERNEL)
    runs = "\n".join(f"    run<{n}, {'true' if rs else 'false'}>(wgs, iters, sms);"
                     for n in NS for rs in (False, True))
    parts.append(HOST.replace("RUNS", runs))
    return "\n".join(parts)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as err:  # noqa: BLE001
        return {"error": str(err)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=4096, help="commit groups per warpgroup (even)")
    ap.add_argument("--json", default=None, help="also write the result to this file")
    ap.add_argument("--compile-only", action="store_true", help="build the program and stop")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        src, exe = os.path.join(tmp, "wgmma_forms.cu"), os.path.join(tmp, "wgmma_forms")
        with open(src, "w") as fp:
            fp.write(source())
        subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        src, "-o", exe], check=True)
        if args.compile_only:
            print("compiled")
            return
        out = subprocess.run([exe, str(args.iters)], capture_output=True, text=True, check=True)
    rows = [json.loads(line) for line in out.stdout.splitlines() if line.strip()]
    for r in rows:
        if "clk_per_mma" in r:
            r["tensor_share"] = r["ideal_clk_per_mma"] / r["clk_per_mma"]
    text = json.dumps({"card": card(), "iters": args.iters, "group": GROUP, "results": rows},
                      indent=1)
    print(text)
    if args.json:
        with open(args.json, "w") as fp:
            fp.write(text + "\n")


if __name__ == "__main__":
    main()
