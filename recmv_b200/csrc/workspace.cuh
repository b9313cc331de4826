// Caller-allocated workspaces.  Every op that takes one has a single layout function that carves it into the op's
// buffers with a Carve.  The size query measures that function on a null base and the run calls it on the caller's
// workspace, so the size and the pointers come from the same code and cannot disagree.
#pragma once
#include <stddef.h>

namespace recmv {

struct Carve {
  char* base;        // nullptr: measure only
  size_t used = 0;   // bytes taken so far

  // The next count elements of T, padded to a multiple of align bytes (a power of two); nullptr when measuring.
  template <class T>
  T* take(size_t count, size_t align = 256) {
    T* p = base ? (T*)(base + used) : nullptr;
    used += (count * sizeof(T) + align - 1) & ~(align - 1);
    return p;
  }
};

// The bytes layout(c, args...) takes: the size query.
template <class Layout, class... Args>
size_t layout_bytes(Layout layout, Args... args) {
  Carve c{nullptr};
  layout(c, args...);
  return c.used;
}

// The buffers layout(c, args...) carves from the workspace at base: the run.
template <class Layout, class... Args>
auto carve(void* base, Layout layout, Args... args) {
  Carve c{(char*)base};
  return layout(c, args...);
}

}  // namespace recmv
