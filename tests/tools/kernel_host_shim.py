"""Compile the device code of the bit-exact kernels — swapnet_b200/csrc/augment.cu (`build`) and csrc/roi_align.cu
(`build_roi`) — and csrc/reflect_pad.h (`build_reflect`) for the HOST (g++, -ffp-contract=off) so that the CPU suite can run the kernel's own source — index arithmetic, pass ping-pong, the IEEE double/float sequence — against the oracle
without a GPU.  Test infrastructure only: the CUDA qualifiers and the round-to-nearest intrinsics are defined away,
blockIdx/threadIdx are globals that a plain loop nest walks.  Nothing in the product uses this."""
import ctypes as C
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PRELUDE = r'''
#include <cstdint>
#include <cmath>
#include <algorithm>
#include "%s/include/swapnet_b200.h"
#define __global__
#define __device__
#define __forceinline__ inline
#define __launch_bounds__(x)
#define __restrict__
struct D3 { int x, y, z; };
static D3 blockIdx, threadIdx, blockDim, gridDim;
using std::min; using std::max;
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline double __dsub_rn(double a, double b) { return a - b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __double2float_rn(double a) { return (float)a; }
'''

DRIVER = r'''
extern "C" void run(const uint8_t* labels, const float* dense, int n, int c, int h, int w, const sn_aug_op* ops,
                    int stride, int max_ops, float* out, float* tmp) {
  AugArgs a; a.labels = labels; a.dense = dense; a.ops = ops; a.out = out; a.tmp = tmp;
  a.n = n; a.c = c; a.h = h; a.w = w; a.stride = stride;
  const int gx = (h + kAugRows - 1) / kAugRows;
  const int passes = max_ops > 0 ? max_ops : 1;
  blockDim = {256, 1, 1}; gridDim = {gx, n * c, 1};
  for (int j = 0; j < passes; ++j) {
    a.pass = j;
    for (int by = 0; by < n * c; ++by) for (int bx = 0; bx < gx; ++bx) for (int t = 0; t < 256; ++t) {
      blockIdx = {bx, by, 0}; threadIdx = {t, 0, 0};
      augment_pass_kernel(a);
    }
  }
}
'''


def build(workdir: str):
    """-> ctypes handle with run(labels, dense, n, c, h, w, ops, stride, max_ops, out, tmp), or None without g++."""
    gxx = shutil.which("g++")
    if gxx is None:
        return None
    src = open(os.path.join(ROOT, "swapnet_b200", "csrc", "augment.cu")).read()
    body = src[src.index("namespace {"):src.index("}  // namespace") + len("}  // namespace")]
    cpp, so = os.path.join(workdir, "augment_host.cpp"), os.path.join(workdir, "libaugment_host.so")
    with open(cpp, "w") as f:
        f.write(PRELUDE % ROOT + body + DRIVER)
    subprocess.run([gxx, "-O1", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, cpp], check=True)
    lib = C.CDLL(so)
    lib.run.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                        C.c_void_p, C.c_void_p]
    lib.run.restype = None
    return lib


ROI_PRELUDE = r'''
#include <cstdint>
#include <cmath>
#include <algorithm>
#define __global__
#define __device__
#define __forceinline__ inline
struct D3 { long long x, y, z; };
static D3 blockIdx, threadIdx, blockDim, gridDim;
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline void split16(float, int, uint16_t& h, uint16_t& l) { h = l = 0; }   // the operand-plane output is not exercised
'''

ROI_DRIVER = r'''
extern "C" void run_roi(const float* tex, int b, int ch, int h, int w, const float* rois, int nroi, int pool, float* out) {
  RoiArgs a; a.tex = tex; a.B = b; a.CH = ch; a.H = h; a.W = w; a.rois = rois; a.nroi = nroi; a.pool = pool;
  a.out = out; a.out_pitch = ch * nroi; a.hi = nullptr; a.lo = nullptr; a.ppitch = 0; a.pcoff = 0; a.fmt = 0;
  blockDim = {1, 1, 1}; gridDim = {1, 1, 1}; blockIdx = {0, 0, 0}; threadIdx = {0, 0, 0};
  roi_align_pack_kernel(a);          // one "thread" walks the whole grid-stride loop
}
'''


def build_roi(workdir: str):
    """csrc/roi_align.cu's device code for the host -> run_roi(tex, b, ch, h, w, rois, nroi, pool, out[b,pool,pool,ch*nroi])."""
    gxx = shutil.which("g++")
    if gxx is None:
        return None
    src = open(os.path.join(ROOT, "swapnet_b200", "csrc", "roi_align.cu")).read()
    body = src[src.index("namespace {"):src.index("}  // namespace") + len("}  // namespace")]
    cpp, so = os.path.join(workdir, "roi_host.cpp"), os.path.join(workdir, "libroi_host.so")
    with open(cpp, "w") as f:
        f.write(ROI_PRELUDE + body + ROI_DRIVER)
    subprocess.run([gxx, "-O1", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, cpp], check=True)
    lib = C.CDLL(so)
    lib.run_roi.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    lib.run_roi.restype = None
    return lib


REFLECT_DRIVER = r'''
#include "%s/swapnet_b200/csrc/reflect_pad.h"
extern "C" int count(int i, int n) { return reflect_pad1_count(i, n); }
extern "C" int position(int i, int n, int k) { return reflect_pad1_position(i, n, k); }
'''


def build_reflect(workdir: str):
    """csrc/reflect_pad.h (the ReflectionPad2d(1) fan-out of the norm/activation kernels) for the host ->
    count(i, n) and position(i, n, k)."""
    gxx = shutil.which("g++")
    if gxx is None:
        return None
    cpp, so = os.path.join(workdir, "reflect_host.cpp"), os.path.join(workdir, "libreflect_host.so")
    with open(cpp, "w") as f:
        f.write(REFLECT_DRIVER % ROOT)
    subprocess.run([gxx, "-O1", "-shared", "-fPIC", "-o", so, cpp], check=True)
    lib = C.CDLL(so)
    lib.count.argtypes = [C.c_int, C.c_int]
    lib.position.argtypes = [C.c_int, C.c_int, C.c_int]
    lib.count.restype = lib.position.restype = C.c_int
    return lib
