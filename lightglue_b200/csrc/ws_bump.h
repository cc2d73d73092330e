// Bump allocator of the workspace carvers (plain C++: the host emulators under oracle/ compile it with g++).
// Each buffer starts at the next multiple of `align` bytes from `base`; with a null base nothing is written and only the
// offsets advance, so one carve function both sizes a workspace (the *_workspace_bytes entry points) and lays it out.
#pragma once
#include <stddef.h>
#include <stdint.h>

struct WsBump {
  char* base;
  size_t off;
  size_t last = 0;  // bytes of the most recent buffer (the layout exports report it)
  template <class T>
  T* take(size_t n, size_t align = 256) {  // align: a power of two
    off = (off + align - 1) & ~(align - 1);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    last = n * sizeof(T);
    off += last;
    return p;
  }
  size_t bytes() const { return (off + 255) & ~(size_t)255; }
};
// The base the layout exports carve from: a carver only forms pointers from its base and never dereferences them, and
// a null base yields null pointers, so the offsets are read as the pointers' distances from this one.
constexpr uintptr_t kLayoutBase = uintptr_t{1} << 20;
