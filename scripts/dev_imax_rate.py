"""Issue rate of the max instructions the kNN sweep's examination is made of, per SM: FMNMX (float max), VIMNMX (integer
max) and VIMNMX3 (Hopper's three-input integer max, __vimax3_s32), next to FADD as the full-rate yardstick.

Compiles a small CUDA program for sm_90a into a temporary directory and runs it: one block of 1024 threads per SM (eight
warps per scheduler), every thread issues batches of 16 independent instructions of one kind; block 0's clock64() span
gives instructions per clock per SM.  --sass prints the opcode counts of the timed loops instead (no GPU needed).  Prints
the card name and its power limit: the numbers mean nothing without them.

    python scripts/dev_imax_rate.py [--sass]
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
SRC = r"""
#include <cstdio>
#include <cuda_runtime.h>
constexpr int ITER = 4096, W = 16;
struct Fadd   { using T = float; static __device__ T op(T a, T b, T c) { return a + b; } };
struct Fmnmx  { using T = float; static __device__ T op(T a, T b, T c) { return fmaxf(a, b); } };
struct Vimnmx { using T = int;   static __device__ T op(T a, T b, T c) { return max(a, b); } };
struct Vimnmx3{ using T = int;   static __device__ T op(T a, T b, T c) { return __vimax3_s32(a, b, c); } };
template <class O>
__global__ void __launch_bounds__(1024, 1) rate(const typename O::T* in, typename O::T* out, long long* span) {
  using T = typename O::T;
  T x[W];
#pragma unroll
  for (int j = 0; j < W; ++j) x[j] = in[threadIdx.x * W + j];
  __syncthreads();
  const long long t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < ITER; ++i) {
    const T c = (T)i;
#pragma unroll
    for (int j = 0; j < W; ++j) x[j] = O::op(x[j], x[(j + 1) % W], c);
  }
  const long long t1 = clock64();
  T s = x[0];
#pragma unroll
  for (int j = 1; j < W; ++j) s = O::op(s, x[j], x[j]);
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (blockIdx.x == 0) { atomicMin(&span[0], t0); atomicMax(&span[1], t1); }
}
template <class O>
void run(const char* name, int sms) {
  typename O::T *in, *out;
  long long* span;
  cudaMalloc(&in, 1024 * W * 4); cudaMemset(in, 0, 1024 * W * 4);
  cudaMalloc(&out, (size_t)sms * 1024 * 4);
  cudaMallocManaged(&span, 16);
  for (int rep = 0; rep < 3; ++rep) {   // the last repetition counts
    span[0] = 0x7fffffffffffffffll; span[1] = 0;
    rate<O><<<sms, 1024>>>(in, out, span);
    if (cudaDeviceSynchronize() != cudaSuccess) { printf("%s: launch failed\n", name); return; }
  }
  printf("%-8s %6.1f instructions / clock / SM  (%lld clocks for %d x %d per thread, 1024 threads)\n", name,
         1024.0 / 32.0 * ITER * W / (double)(span[1] - span[0]), span[1] - span[0], ITER, W);
  cudaFree(in); cudaFree(out); cudaFree(span);
}
int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  run<Fadd>("FADD", p.multiProcessorCount); run<Fmnmx>("FMNMX", p.multiProcessorCount);
  run<Vimnmx>("VIMNMX", p.multiProcessorCount); run<Vimnmx3>("VIMNMX3", p.multiProcessorCount);
  return 0;
}
"""


def card():
    try:
        q = "name,power.limit,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception as exc:
        return f"unknown ({exc!r})"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--sass", action="store_true", help="count the opcodes of the timed loops, run nothing")
    a = p.parse_args()
    with tempfile.TemporaryDirectory(prefix="imax_rate_") as tmp:
        src, exe = os.path.join(tmp, "rate.cu"), os.path.join(tmp, "rate")
        with open(src, "w") as f:
            f.write(SRC)
        arch = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17"]
        if a.sass:
            cubin = os.path.join(tmp, "rate.cubin")
            subprocess.run([os.path.join(CUDA, "bin", "nvcc"), *arch, "-cubin", "-o", cubin, src], check=True)
            sass = subprocess.run([os.path.join(CUDA, "bin", "cuobjdump"), "-sass", cubin], capture_output=True, text=True, check=True).stdout
            for fn in sass.split("Function :")[1:]:
                ops = collections.Counter(re.findall(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_]+)", fn))
                print(fn.split()[0], {k: ops[k] for k in ("FADD", "FMNMX", "VIMNMX", "VIMNMX3", "BRA") if ops[k]})
            return
        subprocess.run([os.path.join(CUDA, "bin", "nvcc"), *arch, "-o", exe, src], check=True)
        print("card:", card(), flush=True)
        sys.stdout.write(subprocess.run([exe], capture_output=True, text=True, check=True).stdout)
        print("card:", card(), flush=True)


if __name__ == "__main__":
    main()
