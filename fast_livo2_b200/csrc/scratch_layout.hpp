// scratch_layout.hpp — how one call's sub-arrays are laid out in a shared per-call block: the device scratch of esikf_ctx
// (esikf_api.cuh) and the pinned host blocks of the shim managers (fl2_shim.cpp).
#pragma once
#include <cstddef>
#include <cstdint>

// One call's scratch block: `lay` takes each sub-array of the call from a ScratchLayout, 256-byte aligned. It runs once with
// base 0 to size the block and, after the one reserve (which discards the old contents), again to hand out the pointers.
struct ScratchLayout {
  uintptr_t base = 0;
  size_t bytes = 0;
  template <typename T> T *take(size_t n) {
    T *p = reinterpret_cast<T *>(base + bytes);
    bytes += (n * sizeof(T) + 255) & ~(size_t)255;
    return p;
  }
};
