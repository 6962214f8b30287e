// Host-side helpers shared by the translation units of the library: device buffers that own their memory and only ever grow,
// fp16-split plane pairs, the kernel launcher, the runtime every handle shares -- its error message, host weights, launch count
// and profiling timeline -- and the error message and argument checks of the calls without a handle.
#pragma once
#include <cstdarg>
#include <cstdio>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/onepose_b200.h"
#include "common.cuh"
#include "gemm_tc.cuh"

namespace opb {

// >= 0: byte value written into every fresh allocation that the algorithm does not require to be zero (opb_debug_set_ws_fill)
int ws_fill_byte();

// Frees its memory on destruction; the owner orders that after the work in flight that may still read it.
struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  bool grew = false;      // set by ensure() when it (re)allocated: the caller orders the fill against its stream
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), bytes(std::exchange(o.bytes, 0)), grew(o.grew) {}
  ~DevBuf() {
    if (p) cudaFree(p);
  }
  cudaError_t ensure(size_t need, bool zero = false) {
    if (need <= bytes) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
    cudaError_t e = cudaMalloc(&p, need);
    if (e != cudaSuccess) return e;
    bytes = need;
    grew = true;
    if (zero) e = cudaMemset(p, 0, need);                                 // buffers whose untouched parts are read as zero (bd, flags)
    else if (ws_fill_byte() >= 0) e = cudaMemset(p, ws_fill_byte(), need);   // test hook: poison everything else
    return e;
  }
  template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

// A window of rows of a [rows, 256] plane pair (the residual stream of a chunk, the query-only buffer, ...).
struct XView {
  __half* hi;
  __half* lo;
  CPlanes c(int ld) const { return CPlanes{hi, lo, ld}; }
  Planes m(int ld) const { return Planes{hi, lo, ld}; }
};

struct PlaneBuf {
  DevBuf hi, lo;
  cudaError_t ensure(size_t elems, bool zero = false) {
    cudaError_t e = hi.ensure(elems * sizeof(__half), zero);
    if (e != cudaSuccess) return e;
    return lo.ensure(elems * sizeof(__half), zero);
  }
  CPlanes c(int ld, size_t off_elems = 0) const { return CPlanes{hi.as<__half>() + off_elems, lo.as<__half>() + off_elems, ld}; }
  Planes m(int ld, size_t off_elems = 0) const { return Planes{hi.as<__half>() + off_elems, lo.as<__half>() + off_elems, ld}; }
  XView view(size_t row_off = 0) const { return XView{hi.as<__half>() + row_off * kD, lo.as<__half>() + row_off * kD}; }
};

inline void split_host(const std::vector<double>& w, std::vector<__half>& hi, std::vector<__half>& lo) {
  hi.resize(w.size());
  lo.resize(w.size());
  for (size_t i = 0; i < w.size(); ++i) split_f32((float)w[i], hi[i], lo[i]);
}

// `pdl`: launch with programmatic stream serialization (PDL).  Only a kernel that begins with griddep_sync() may take it: the
// handles' launches pass pdl_enabled(), and a kernel that reads its inputs without that wait is launched without it.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(bool pdl, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

// Profile of the counted launches of a handle's last forward (bench.py roofline legs): with profiling on, a start event and
// one event after every launch on its stream.  Entry i's time is its event minus the one before (the start event for entry 0),
// so it includes any launch gap in front of it.
struct Timeline {
  bool on = false;
  cudaEvent_t start = nullptr;
  cudaEvent_t end = nullptr;           // recorded by finish(): the matcher's forward spans start .. end
  std::vector<cudaEvent_t> ev;         // pool: entry i is recorded on ev[i]
  std::vector<std::string> name;
  std::vector<double> flops;           // algorithmic FLOPs of each entry (0 for the helper kernels)
  Timeline() = default;
  Timeline(const Timeline&) = delete;
  Timeline& operator=(const Timeline&) = delete;
  ~Timeline() {
    for (cudaEvent_t e : ev) cudaEventDestroy(e);
    if (start) cudaEventDestroy(start);
    if (end) cudaEventDestroy(end);
  }
  size_t size() const { return name.size(); }
  void clear() {
    name.clear();
    flops.clear();
  }
  void begin(cudaStream_t st) {
    clear();
    if (on) cudaEventRecord(event(start), st);
  }
  void mark(cudaStream_t st, const char* n, double f) {
    if (!on) return;
    if (ev.size() == name.size()) ev.push_back(nullptr);
    cudaEventRecord(event(ev[name.size()]), st);
    name.push_back(n);
    flops.push_back(f);
  }
  void finish(cudaStream_t st) {
    if (on) cudaEventRecord(event(end), st);
  }
  cudaError_t ms(size_t i, float* t) const { return cudaEventElapsedTime(t, i ? ev[i - 1] : start, ev[i]); }

 private:
  static cudaEvent_t event(cudaEvent_t& e) {
    if (!e) cudaEventCreate(&e);
    return e;
  }
};

// Makes `device` the current device for the guard's lifetime and gives the caller's current device back afterwards.  Every
// entry point of a handle runs under one, so a handle's work lands on its own device whatever device the caller has current.
struct DeviceGuard {
  int prev = -1;                 // caller's device to restore; -1: nothing to restore
  cudaError_t err = cudaSuccess;
  explicit DeviceGuard(int device) {
    int cur = 0;
    err = cudaGetDevice(&cur);
    if (err == cudaSuccess && cur != device) {
      err = cudaSetDevice(device);
      if (err == cudaSuccess) prev = cur;
    }
  }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// State every handle of the library has; opb_matcher and opb_superpoint derive from it.
struct Handle {
  std::string err;                                     // message of the last failed call (opb_last_error / opb_sp_last_error)
  std::map<std::string, std::vector<float>> host_w;    // weights as loaded, by name
  int find_code = 0;                                   // code of the last failed find_weight
  int launches = 0;                                    // counted launches since begin()
  Timeline timeline;
  int device = 0;                                      // the handle's device: its memory lives there and its work runs there
  // Calls of one handle share its workspace and object buffers, so they are ordered across the caller's streams: every call that
  // enqueues work records `ev` on its stream when it ends (enqueued()), and a call on another stream first makes its stream wait
  // for that event (enter()) -- a device-side wait, the host does not block.  `ev` also tells when the last call has finished
  // (the range reports wait for it).
  cudaEvent_t ev = nullptr;
  cudaStream_t ev_stream = nullptr;                    // stream `ev` was last recorded on
  bool ev_recorded = false;
  Handle() = default;
  Handle(const Handle&) = delete;
  Handle& operator=(const Handle&) = delete;
  ~Handle() {
    if (ev) cudaEventDestroy(ev);
  }
  cudaError_t enter(cudaStream_t st) const { return ev_recorded && st != ev_stream ? cudaStreamWaitEvent(st, ev, 0) : cudaSuccess; }
  cudaError_t enqueued(cudaStream_t st) {
    ev_stream = st;
    ev_recorded = true;
    return cudaEventRecord(ev, st);
  }
  // Host-side wait for the last call (before host copies that overwrite buffers it may still read).
  cudaError_t drain() const { return ev_recorded ? cudaEventSynchronize(ev) : cudaSuccess; }
  void begin(cudaStream_t st) {
    launches = 0;
    timeline.begin(st);
  }
  void counted(cudaStream_t st, const char* name, double flops) {
    launches++;
    timeline.mark(st, name, flops);
  }
};

// The message of the last failed call on this thread that had no handle (the create functions and the handle-free entry
// points): what opb_last_error(NULL) and opb_sp_last_error(NULL) return.  A successful call leaves it as it is.
inline thread_local std::string no_handle_error;

// Sets the message of a failed call and returns its code: into the handle, or -- for a call that has none -- into
// no_handle_error.
inline void set_error(std::string& dst, const char* fmt, va_list ap) {
  char buf[512];
  vsnprintf(buf, sizeof buf, fmt, ap);
  dst = buf;
}
inline int fail(std::string& dst, int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  set_error(dst, fmt, ap);
  va_end(ap);
  return code;
}
inline int fail(Handle* h, int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  set_error(h->err, fmt, ap);
  va_end(ap);
  return code;
}

#define CK(h, expr)                                                                                   \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess)                                                                            \
      return opb::fail(h, OPB_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// Runs `enqueue()` -- the part of a call that enqueues work for handle `h` on `st` -- after the handle's previous call, and
// records the handle's event behind it (Handle::enter / enqueued).
template <typename F>
inline int ordered(Handle* h, cudaStream_t st, F&& enqueue) {
  CK(h, h->enter(st));
  const int rc = enqueue();
  const cudaError_t e = h->enqueued(st);
  if (rc) return rc;
  CK(h, e);
  return OPB_OK;
}

// Result of a counted launch of kernel `name`: a failure becomes the handle's error, a success is counted and profiled.
inline int launched(Handle* h, cudaStream_t st, const char* name, cudaError_t e) {
  if (e != cudaSuccess) return fail(h, OPB_E_CUDA, "launch of %s failed: %s", name, cudaGetErrorString(e));
  h->counted(st, name, 0.0);
  return 0;
}

#define LAUNCH(h, st, name, ...)                                                            \
  do {                                                                                      \
    if (int _rc = launched(h, st, name, launch_k(pdl_enabled(), __VA_ARGS__))) return _rc; \
  } while (0)

// Argument check of entry point `fn` without a handle: OPB_E_INVALID unless `cond` holds, with a message that names both.
#define REQUIRE(fn, cond) \
  do { if (!(cond)) return opb::fail(opb::no_handle_error, OPB_E_INVALID, "%s: %s", fn, #cond); } while (0)

// Result of the launch of kernel `name` by entry point `fn` without a handle: a failure becomes OPB_E_CUDA and the message.
inline int launched(const char* fn, const char* name, cudaError_t e) {
  return e == cudaSuccess ? OPB_OK : fail(no_handle_error, OPB_E_CUDA, "%s: launch of %s failed: %s", fn, name, cudaGetErrorString(e));
}

// A launch by entry point `fn` without a handle.  Its kernels do not begin with griddep_sync(), so they go without PDL.
#define LAUNCH_NH(fn, kern, ...) \
  do { if (int _rc = opb::launched(fn, #kern, opb::launch_k(false, kern, __VA_ARGS__))) return _rc; } while (0)

// One counted launch of the wgmma GEMM core: `flops` = algorithmic FLOPs, `name` = its profile entry, `what` names it in an error.
inline int run_gemm(Handle* h, const GemmProblem& p, cudaStream_t st, double flops, const char* what, const char* name) {
  const int rc = launch_gemm_tc(p, st);
  h->counted(st, name, flops);
  if (rc != 0)
    return fail(h, rc == -1 ? OPB_E_INVALID : OPB_E_CUDA, "GEMM launch failed (%s, rc=%d): %s", what, rc, cudaGetErrorString(cudaGetLastError()));
  return 0;
}

// A loaded weight of `n` elements; otherwise null, with the message and find_code set (OPB_E_STATE: missing, OPB_E_INVALID:
// wrong size).  The finalize functions look up a group of weights and then return find_code.
inline const std::vector<float>* find_weight(Handle* h, const std::string& key, size_t n) {
  auto it = h->host_w.find(key);
  if (it == h->host_w.end()) {
    h->find_code = fail(h, OPB_E_STATE, "missing weight '%s'", key.c_str());
    return nullptr;
  }
  if (it->second.size() != n) {
    h->find_code = fail(h, OPB_E_INVALID, "weight '%s' has %zu elements, expected %zu", key.c_str(), it->second.size(), n);
    return nullptr;
  }
  return &it->second;
}

// Weight uploads are synchronous copies on the legacy stream; the finalize functions end with a device synchronisation so that
// they are ordered against whatever (non-blocking) stream the caller uses afterwards.
// `w` as fp16-split planes at element `off_elems` of `dst`, which holds `total_elems` (0: w.size()).
inline int upload_planes(Handle* h, PlaneBuf& dst, const std::vector<double>& w, size_t off_elems = 0, size_t total_elems = 0) {
  std::vector<__half> hi, lo;
  split_host(w, hi, lo);
  CK(h, dst.ensure(total_elems ? total_elems : w.size()));
  CK(h, cudaMemcpy(dst.hi.as<__half>() + off_elems, hi.data(), hi.size() * sizeof(__half), cudaMemcpyHostToDevice));
  CK(h, cudaMemcpy(dst.lo.as<__half>() + off_elems, lo.data(), lo.size() * sizeof(__half), cudaMemcpyHostToDevice));
  return 0;
}
inline int upload_f32(Handle* h, DevBuf& dst, const std::vector<double>& w) {
  std::vector<float> f(w.begin(), w.end());
  CK(h, dst.ensure(f.size() * sizeof(float)));
  CK(h, cudaMemcpy(dst.p, f.data(), f.size() * sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

// create: `device` must be an sm_90 device; `prop` receives its properties.  The caller's current device is left as it is (the
// create functions make `device` current with a DeviceGuard).  Messages go to `err`.
inline int select_device(int device, cudaDeviceProp& prop, std::string& err) {
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0) return fail(err, OPB_E_CUDA, "no CUDA device: %s (this library has no CPU path)", cudaGetErrorString(e));
  if (device < 0 || device >= n_dev) return fail(err, OPB_E_INVALID, "device %d out of range", device);
  e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) return fail(err, OPB_E_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
  if (prop.major != 9 || prop.minor != 0)
    return fail(err, OPB_E_CUDA, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
  return OPB_OK;
}

// The rest of a handle's creation on its (already current) device: the order event and the pinned copy of the range flag.
inline int create_handle_state(Handle* h, int device, int** range_host, std::string& err) {
  h->device = device;
  if (cudaMallocHost(range_host, sizeof(int)) != cudaSuccess || cudaEventCreateWithFlags(&h->ev, cudaEventDisableTiming) != cudaSuccess)
    return fail(err, OPB_E_CUDA, "pinned flag / event allocation failed");
  **range_host = 0;
  return OPB_OK;
}

#ifdef __CUDACC__
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
#endif

}  // namespace opb
