// hwy_abi.h — error reporting / launch counting / launch set-up shared by the library's translation units.
// Every function returns 0, or 1 after setting hwy_last_error().
#pragma once
#include <cstddef>

namespace hwy_abi {
int fail(const char* fmt, const char* detail);   // sets hwy_last_error(), returns 1
int check_launch(const char* what);              // counts the launch, returns 1 on a CUDA error

int require_device();                            // a CUDA device exists: the library has no CPU fallback
int current_device(int& dev);                    // the calling thread's device, 0..63
struct DeviceProps {
    int n_sm, smem_sm, smem_block;               // SMs, shared memory per SM, opt-in shared memory per block
};
int device_props(DeviceProps& out);              // of the current device, queried once per device
// Raises the dynamic shared memory limit of `kernel` (a __global__ function) on the current device to `bytes`, unless
// an earlier call already raised it that far.
int opt_in_smem(const void* kernel, size_t bytes);
}  // namespace hwy_abi
