// pack.h -- lays out a solver's arrays in one device block, with a host mirror for the ones the host fills (pure host C++, so
// that the CPU emulation harness builds the solvers' packers without CUDA headers)
//
// A packer names each array once: one `put` (inputs: reserved, and copied into the mirror) or `take` (work and outputs: reserved
// only) returns the array's device address.  Like carve_scratch (scratch.h), it runs twice: with a null device base to measure,
// then on the allocated block.
#pragma once
#include <assert.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

namespace orb {

struct PackRegion {
    uint8_t* dev;    // device address of the region's first byte; nullptr: measure only
    uint8_t* host;   // mirror of the region (nullptr for a region that is only reserved)
    size_t align;    // every array starts at a multiple of this
    size_t off = 0;

    // n elements, plus `spare` never written (an empty array still gets an address of its own)
    template <typename T>
    T* take(size_t n, size_t spare = 0) {
        off = (off + align - 1) / align * align;
        T* p = dev ? reinterpret_cast<T*>(dev + off) : nullptr;
        off += (n + spare) * sizeof(T);
        return p;
    }
    template <typename T>
    T* put(const T* src, size_t n, size_t spare = 0) {
        T* p = take<T>(n, spare);
        if (p && n) {
            assert(host);
            memcpy(host + (reinterpret_cast<uint8_t*>(p) - dev), src, n * sizeof(T));
        }
        return p;
    }
    size_t bytes() const { return (off + align - 1) / align * align; }
};

}  // namespace orb
