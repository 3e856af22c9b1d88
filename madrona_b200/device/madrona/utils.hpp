// Reference: include/madrona/utils.hpp (subset used by simulators).
#pragma once
#include <madrona/types.hpp>
#include <madrona/span.hpp>
namespace madrona {

// Ring buffer over caller storage (reference: utils.hpp:64-83, utils.inl:3-53).  It holds
// at most capacity - 1 elements: head == tail means empty.
template <typename T>
class ArrayQueue {
public:
    MB2_HD inline ArrayQueue(T *data, uint32_t capacity)
        : data_(data), capacity_(capacity), head_(0), tail_(0) {}

    MB2_HD inline void add(T t)
    {
        data_[tail_] = t;
        tail_ = increment(tail_);
    }

    MB2_HD inline T remove()
    {
        T t = data_[head_];
        head_ = increment(head_);
        return t;
    }

    MB2_HD inline uint32_t capacity() const { return capacity_; }
    MB2_HD inline bool isEmpty() const { return head_ == tail_; }
    MB2_HD inline void clear() { head_ = 0; tail_ = 0; }

private:
    MB2_HD inline uint32_t increment(uint32_t i) { return i == capacity_ - 1 ? 0 : i + 1; }

    T *data_;
    uint32_t capacity_;
    uint32_t head_;
    uint32_t tail_;
};

namespace utils {
template <typename T> struct TypeIdentity { using type = T; };
template <typename T> using TypeIdentityT = typename TypeIdentity<T>::type;

template <typename T>
MB2_HD constexpr inline T divideRoundUp(T a, T b) { return (a + (b - 1)) / b; }
template <typename T>
MB2_HD constexpr inline T roundUp(T v, T mult) { return divideRoundUp(v, mult) * mult; }
MB2_HD constexpr inline uint64_t roundUpPow2(uint64_t v, uint64_t p) { return (v + p - 1) & ~(p - 1); }
// alignment must be a power of 2
MB2_HD inline uintptr_t alignPtrOffset(void *ptr, uintptr_t alignment)
{
    uintptr_t base = (uintptr_t)ptr;
    return (uintptr_t)roundUpPow2(base, alignment) - base;
}
MB2_HD inline void *alignPtr(void *ptr, uintptr_t alignment)
{
    return (char *)ptr + alignPtrOffset(ptr, alignment);
}
// Both overloads say 0 is not a power of 2 (the reference says it is; nothing relies on it).
MB2_HD constexpr inline bool isPower2(uint64_t v) { return v && !(v & (v - 1)); }
MB2_HD constexpr inline bool isPower2(uint32_t v) { return v && !(v & (v - 1)); }
MB2_HD constexpr inline uint32_t u32mulhi(uint32_t a, uint32_t b)
{
    return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
}
MB2_HD constexpr inline uint32_t int32NextPow2(uint32_t v)
{
    v--; v |= v >> 1; v |= v >> 2; v |= v >> 4; v |= v >> 8; v |= v >> 16;
    return v + 1;
}
MB2_HD constexpr inline uint64_t int64NextPow2(uint64_t v)
{
    v--; v |= v >> 1; v |= v >> 2; v |= v >> 4; v |= v >> 8; v |= v >> 16; v |= v >> 32;
    return v + 1;
}
MB2_HD constexpr inline uint32_t int32Log2(uint32_t v) { return 31u - (uint32_t)MB2_CLZ(v); }
MB2_HD constexpr inline uint64_t int64Log2(uint64_t v) { return 63u - (uint64_t)MB2_CLZLL(v); }
// lowbias32 of the hash-prospector (C. Wellons): the same bits as the reference's int32Hash
MB2_HD constexpr inline uint32_t int32Hash(uint32_t x)
{
    x ^= x >> 16u;
    x *= 0x7feb352du;
    x ^= x >> 15u;
    x *= 0x846ca68bu;
    x ^= x >> 16u;
    return x;
}
// Offsets of chunks 1 .. n-1 packed after chunk 0, each at pow2_alignment; returns the
// total, rounded up to the alignment
MB2_HD inline int64_t computeBufferOffsets(const Span<const int64_t> chunk_sizes,
                                           Span<int64_t> out_offsets,
                                           int64_t pow2_alignment)
{
    int64_t total = chunk_sizes[0];
    for (CountT i = 1; i < chunk_sizes.size(); i++) {
        int64_t off = (int64_t)roundUpPow2((uint64_t)total, (uint64_t)pow2_alignment);
        out_offsets[i - 1] = off;
        total = off + chunk_sizes[i];
    }
    return (int64_t)roundUpPow2((uint64_t)total, (uint64_t)pow2_alignment);
}
template <typename T>
MB2_HD inline void copyN(TypeIdentityT<T> *dst, const TypeIdentityT<T> *src, CountT num_elems)
{
    for (CountT i = 0; i < num_elems; i++) dst[i] = src[i];
}
template <typename T>
MB2_HD inline void zeroN(TypeIdentityT<T> *ptr, CountT num_elems)
{
    for (CountT i = 0; i < num_elems; i++) ptr[i] = T {};
}
template <typename T>
MB2_HD inline void fillN(TypeIdentityT<T> *ptr, T v, CountT num_elems)
{
    for (CountT i = 0; i < num_elems; i++) ptr[i] = v;
}
template <typename T> MB2_HD constexpr inline T clamp(T v, T lo, T hi) { return v < lo ? lo : (v > hi ? hi : v); }
}
}
