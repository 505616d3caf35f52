// Host-side plumbing shared by the eight C-ABI modules (lspg, lsph, lspm, lspa, lspl, lspr, lspj, lspv): the per-module error
// channel, device validation, the current-device guard and the state-dict table.  No device code.
//
// Each module binds the error channel to a tag type of its own in one line,
//   struct Lspx;  constexpr auto fail = capi::fail<Lspx>;
// so lspx_last_error() reports the last failed lspx_* call on the calling thread, whatever other modules did since.
#pragma once

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <map>
#include <string>

#include "../../include/lspg.h"

namespace capi {

template <class Module>
std::string& last_error() {
  static thread_local std::string message;
  return message;
}

// Records a printf-style message on Module's channel and returns code.
template <class Module>
int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  last_error<Module>() = buf;
  return code;
}

// The `device` argument of every *_create: -1 is a host-only handle; otherwise it must name an sm_90 device, whose
// properties land in *prop.
template <class Module>
int check_device(int device, cudaDeviceProp* prop) {
  if (device < -1) return fail<Module>(LSPG_EINVAL, "device must be >= -1 (got %d)", device);
  if (device == -1) return LSPG_OK;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) return fail<Module>(LSPG_ENODEV, "no CUDA device: %s", cudaGetErrorString(e));
  if (device >= count) return fail<Module>(LSPG_ENODEV, "device %d out of range (%d devices)", device, count);
  e = cudaGetDeviceProperties(prop, device);
  if (e != cudaSuccess)
    return fail<Module>(LSPG_ECUDA, "cudaGetDeviceProperties(&prop, device) failed: %s", cudaGetErrorString(e));
  if (prop->major != 9 || prop->minor != 0)
    return fail<Module>(LSPG_ENODEV, "device %d is sm_%d%d; this library contains sm_90a code only (no fallback)", device,
                        prop->major, prop->minor);
  return LSPG_OK;
}

// The refusal of a call that needs the device on a host-only handle.
template <class Module>
int require_device(int device, const char* fn) {
  if (device >= 0) return LSPG_OK;
  return fail<Module>(LSPG_ENODEV, "host-only handle: %s needs an sm_90 device (no CPU path exists)", fn);
}

// Makes `device` current for the scope and restores the caller's device when it ends, so no call leaves the calling
// thread (and torch, which reads it back with cudaGetDevice) on the handle's device.  A host-only handle (device < 0)
// makes no CUDA call.
class DeviceGuard {
 public:
  explicit DeviceGuard(int device) : dev_(device) {
    if (dev_ < 0) return;
    cudaGetDevice(&prev_);
    if (prev_ != dev_) cudaSetDevice(dev_);
  }
  ~DeviceGuard() {
    if (dev_ >= 0 && prev_ != dev_) cudaSetDevice(prev_);
  }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;

 private:
  int dev_, prev_ = 0;
};

// A state dict passed as lspg_tensor[n], by name, with the nn.DataParallel prefix "module." stripped
// (base_model.py:213-215).  After construction, status() is LSPG_OK or the refusal of a null name or data pointer.
template <class Module>
class WeightTable {
 public:
  WeightTable(const lspg_tensor* tensors, int n) {
    for (int i = 0; i < n; ++i) {
      if (!tensors[i].name || !tensors[i].data) {
        rc_ = fail<Module>(LSPG_EINVAL, "tensor %d has a null name or data pointer", i);
        return;
      }
      std::string nm = tensors[i].name;
      if (nm.rfind("module.", 0) == 0) nm = nm.substr(7);
      by_name_[nm] = &tensors[i];
    }
  }

  int status() const { return rc_; }

  const lspg_tensor* find(const std::string& key) const {
    auto it = by_name_.find(key);
    return it == by_name_.end() ? nullptr : it->second;
  }

  // The data of `key` if it is present with `expect` elements, else null.  The first missing required key or wrong
  // element count is recorded, and stays in status().
  const float* get(const std::string& key, size_t expect, bool required = true) {
    const lspg_tensor* t = find(key);
    if (!t) {
      if (required && rc_ == LSPG_OK) rc_ = fail<Module>(LSPG_ESTATE, "missing parameter %s", key.c_str());
      return nullptr;
    }
    if (static_cast<size_t>(t->numel) != expect) {
      if (rc_ == LSPG_OK)
        rc_ = fail<Module>(LSPG_EINVAL, "%s has %lld elements, expected %zu", key.c_str(), static_cast<long long>(t->numel),
                           expect);
      return nullptr;
    }
    return t->data;
  }

 private:
  std::map<std::string, const lspg_tensor*> by_name_;
  int rc_ = LSPG_OK;
};

}  // namespace capi

// Returns LSPG_ECUDA with the failing expression from the enclosing function, on the channel of the translation unit's
// `fail`.
#define CUDA_TRY(expr)                                                                              \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess) return fail(LSPG_ECUDA, "%s failed: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)
