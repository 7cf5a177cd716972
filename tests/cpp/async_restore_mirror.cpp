// Compiles the C++ mirror's decode and Unwrap from device-written offsets (include/lz4net.hpp) against the C ABI
// (include/lz4b200.h): every argument converts as the header declares it.  Compiled only; the GPU tests run the calls.
#include "lz4net.hpp"

void async_restore_mirror(LZ4::Context& ctx, const void* pinned, const int64_t* dev_off, void* dev_dst, const int64_t* dst_off,
                          const int32_t* cap, int32_t* out_len, int32_t n, void* stream)
{
    ctx.decode_from_host_at_async(pinned, 1 << 20, dev_off, dev_dst, dst_off, cap, out_len, n, true, stream);
    ctx.unwrap_from_host_at_async(pinned, 1 << 20, dev_off, dev_dst, dst_off, cap, out_len, n, stream);
}
