// Compiles the C++ mirror's LZ4Stream decode from a device-written size (include/lz4net.hpp) against the C ABI
// (include/lz4b200.h): every argument converts as the header declares it.  Compiled only; the GPU tests run the call.
#include "lz4net.hpp"

void async_stream_restore_mirror(LZ4::Context& ctx, const void* pinned, const int64_t* dev_size, void* dev_dst, int64_t* out_size,
                                 void* stream)
{
    ctx.stream_decode_from_host_at_async(pinned, 1 << 20, dev_size, 65536, dev_dst, 1 << 22, out_size, stream);
}
