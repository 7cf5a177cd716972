// Compiles the C++ mirror's asynchronous LZ4Stream methods (include/lz4net.hpp) against the C ABI (include/lz4b200.h):
// every argument converts as the header declares it.  Compiled only; the GPU tests run the calls.
#include "lz4net.hpp"

void async_stream_mirror(LZ4::Context& ctx, const void* dev_src, void* pinned, void* dev_dst, int64_t n, int64_t* out_size,
                         void* stream)
{
    ctx.stream_encode_to_host_async(dev_src, n, 1 << 16, true, pinned, lz4b200_stream_bound(n, 1 << 16), out_size, stream);
    ctx.stream_decode_from_host_async(pinned, n, dev_dst, n, out_size, stream);
}
