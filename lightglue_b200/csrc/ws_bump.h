// Bump allocator of the workspace carvers (plain C++: the host emulators under oracle/ compile it with g++).
// Each buffer starts at the next multiple of `align` bytes from `base`; with a null base nothing is written and only the
// offsets advance, so one carve function both sizes a workspace (the *_workspace_bytes entry points) and lays it out.
#pragma once
#include <stddef.h>

struct WsBump {
  char* base;
  size_t off;
  template <class T>
  T* take(size_t n, size_t align = 256) {  // align: a power of two
    off = (off + align - 1) & ~(align - 1);
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += n * sizeof(T);
    return p;
  }
  size_t bytes() const { return (off + 255) & ~(size_t)255; }
};
