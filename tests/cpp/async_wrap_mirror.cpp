// Compiles the C++ mirror's asynchronous packed decode, Wrap and Unwrap methods (include/lz4net.hpp) against the C ABI
// (include/lz4b200.h): every argument converts as the header declares it.  Compiled only; the GPU tests run the calls.
#include "lz4net.hpp"

void async_wrap_mirror(LZ4::Context& ctx, const void* dev_src, void* pinned, void* dev_dst, const int64_t* off,
                       const int32_t* len, const int32_t* cap, int64_t* out_off, int32_t* out_len, int32_t n, void* stream)
{
    ctx.decode_packed_from_host_async(pinned, off, len, dev_dst, 1 << 20, out_off, out_len, n, stream);
    ctx.wrap_packed_to_host_async(dev_src, off, len, pinned, 1 << 20, out_off, out_len, n, true, stream);
    ctx.unwrap_from_host_async(pinned, off, len, dev_dst, off, cap, out_len, n, stream);
    ctx.unwrap_packed_from_host_async(pinned, off, len, dev_dst, 1 << 20, out_off, out_len, n, stream);
}
