// lz4net.hpp -- C++ host-side mirror of lz4net's public surface for the accelerated path, header-only over the C ABI
// (include/lz4b200.h).  The reference is compiled code whose toolchain (.NET) is absent here, so this is the host
// layer "above the ABI" in C++: same names, argument meaning and error behaviour as the C# originals.
//
//   LZ4::ILZ4Service / LZ4::CudaLZ4Service   src/LZ4/ILZ4Service.cs:30-36, src/LZ4/Services/CppMM64LZ4Service.cs:31-52
//   LZ4::LZ4Codec                            src/LZ4/LZ4Codec.cs:313-440 (Encode/EncodeHC/Decode), :510-599 (Wrap/Unwrap)
//   LZ4::LZ4Stream                           src/LZ4/LZ4Stream.cs (chunked stream; here K blocks are dispatched per GPU batch)
//
// byte[] + offset + length become (pointer, offset, length); exceptions map to std::invalid_argument (ArgumentException),
// std::runtime_error (EndOfStreamException / NotSupportedException).
#pragma once
#include "lz4b200.h"

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <istream>
#include <ostream>
#include <stdexcept>
#include <string>
#include <vector>

namespace LZ4 {

struct ILZ4Service {                                                     // src/LZ4/ILZ4Service.cs:30-36
    virtual ~ILZ4Service() {}
    virtual std::string CodecName() const = 0;
    virtual int Encode(const uint8_t* input, int inputOffset, int inputLength, uint8_t* output, int outputOffset, int outputLength) = 0;
    virtual int EncodeHC(const uint8_t* input, int inputOffset, int inputLength, uint8_t* output, int outputOffset, int outputLength) = 0;
    virtual int Decode(const uint8_t* input, int inputOffset, int inputLength, uint8_t* output, int outputOffset, int outputLength, bool knownOutputLength) = 0;
};

class CudaLZ4Service : public ILZ4Service {
public:
    CudaLZ4Service() { if (lz4b200_device_count() < 1) throw std::runtime_error("CudaLZ4Service: no sm_90 device"); }
    std::string CodecName() const override { return "CUDA sm_90a"; }
    int Encode(const uint8_t* in, int io, int il, uint8_t* out, int oo, int ol) override
    {
        if (il == 0 || ol == 0) return 0;                                // src/LZ4ps/LZ4Codec.cs:156-160, Safe.cs:403
        return lz4b200_compress_limitedOutput((const char*)in + io, (char*)out + oo, il, ol);
    }
    int EncodeHC(const uint8_t* in, int io, int il, uint8_t* out, int oo, int ol) override
    {
        if (il == 0) return 0;
        if (ol == 0) return -1;
        const int n = lz4b200_compressHC_limitedOutput((const char*)in + io, (char*)out + oo, il, ol);
        return n <= 0 ? -1 : n;                                          // src/LZ4ps/LZ4Codec.Safe.cs:721-723
    }
    int Decode(const uint8_t* in, int io, int il, uint8_t* out, int oo, int ol, bool known) override
    {
        if (il == 0 || ol == 0) return 0;                                // LZ4Codec.cs:156-160, Safe.cs:470
        if (known) {
            if (lz4b200_uncompress((const char*)in + io, (char*)out + oo, il, ol) != il)      // Safe.cs:539-542
                throw std::invalid_argument("LZ4 block is corrupted, or invalid length has been given.");
            return ol;
        }
        const int n = lz4b200_uncompress_unknownOutputSize((const char*)in + io, (char*)out + oo, il, ol);
        if (n < 0) throw std::invalid_argument("LZ4 block is corrupted, or invalid length has been given.");   // :546-549
        return n;
    }
};

class Context {                                                          // owns one lz4b200_ctx (the GPU path has state)
public:
    explicit Context(int device = 0) { if (lz4b200_create(&h_, device) != LZ4B200_OK) throw std::runtime_error(lz4b200_last_error()); }
    ~Context() { lz4b200_destroy(h_); }
    Context(const Context&) = delete; Context& operator=(const Context&) = delete;
    lz4b200_ctx* handle() const { return h_; }
    // What a host-memory decode of these blocks would return per block (bytes written; with known sizes: bytes read), without
    // decoding.  dst_cap may be null for unknown sizes: no limit.
    std::vector<int32_t> measure(const uint8_t* src, const int64_t* src_off, const int32_t* src_len, const int32_t* dst_cap,
                                 int32_t n, bool known = false)
    {
        std::vector<int32_t> out((size_t)std::max(n, 0));
        if (lz4b200_measure_batch(h_, src, src_off, src_len, dst_cap, out.data(), n, known ? 1 : 0, LZ4B200_MEM_HOST, nullptr) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
        return out;
    }
    // Offload without blocking: blocks of device memory encoded back to back into page-locked host memory, and blocks of
    // page-locked host memory decoded into device memory (lz4b200_encode_batch_packed_from_device_async,
    // lz4b200_decode_batch_to_device_async).  Enqueued on `stream`, they return at once; src, dst, out_off and out_len stay
    // the caller's, alive and untouched, until the stream has passed the call.
    void encode_packed_to_host_async(const void* src, const int64_t* src_off, const int32_t* src_len, const int32_t* dst_cap,
                                     void* dst, int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n,
                                     bool hc, void* stream)
    {
        if (lz4b200_encode_batch_packed_from_device_async(h_, src, src_off, src_len, dst_cap, dst, dst_total_cap, out_off, out_len, n,
                                                          hc ? LZ4B200_MODE_HC : LZ4B200_MODE_FAST, stream) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
    }
    void decode_from_host_async(const void* src, const int64_t* src_off, const int32_t* src_len, void* dst, const int64_t* dst_off,
                                const int32_t* dst_cap, int32_t* out_len, int32_t n, bool known, void* stream)
    {
        if (lz4b200_decode_batch_to_device_async(h_, src, src_off, src_len, dst, dst_off, dst_cap, out_len, n, known ? 1 : 0,
                                                 stream) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
    }
    // The same for the packed unknown-size decode and for Wrap packets (lz4b200_decode_batch_packed_to_device_async,
    // lz4b200_wrap_batch_packed_from_device_async, lz4b200_unwrap_batch_to_device_async,
    // lz4b200_unwrap_batch_packed_to_device_async).  The packed forms' out_off (n + 1 entries) is written by the device.
    void decode_packed_from_host_async(const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                                       int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n, void* stream)
    {
        if (lz4b200_decode_batch_packed_to_device_async(h_, src, src_off, src_len, dst, dst_total_cap, out_off, out_len, n,
                                                        stream) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
    }
    void wrap_packed_to_host_async(const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                                   int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n, bool hc, void* stream)
    {
        if (lz4b200_wrap_batch_packed_from_device_async(h_, src, src_off, src_len, hc ? 1 : 0, dst, dst_total_cap, out_off, out_len,
                                                        n, stream) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
    }
    void unwrap_from_host_async(const void* src, const int64_t* src_off, const int32_t* src_len, void* dst, const int64_t* dst_off,
                                const int32_t* dst_cap, int32_t* out_len, int32_t n, void* stream)
    {
        if (lz4b200_unwrap_batch_to_device_async(h_, src, src_off, src_len, dst, dst_off, dst_cap, out_len, n, stream) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
    }
    void unwrap_packed_from_host_async(const void* src, const int64_t* src_off, const int32_t* src_len, void* dst,
                                       int64_t dst_total_cap, int64_t* out_off, int32_t* out_len, int32_t n, void* stream)
    {
        if (lz4b200_unwrap_batch_packed_to_device_async(h_, src, src_off, src_len, dst, dst_total_cap, out_off, out_len, n,
                                                        stream) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
    }
    // The decode and the Unwrap from offsets the device wrote (lz4b200_decode_batch_to_device_at_async,
    // lz4b200_unwrap_batch_to_device_at_async): src_off (n + 1 entries, device or page-locked memory) is read on the device,
    // so the out_off of a packed offload above can be passed straight in; only src_cap bytes of src are read.
    void decode_from_host_at_async(const void* src, int64_t src_cap, const int64_t* src_off, void* dst, const int64_t* dst_off,
                                   const int32_t* dst_cap, int32_t* out_len, int32_t n, bool known, void* stream)
    {
        if (lz4b200_decode_batch_to_device_at_async(h_, src, src_cap, src_off, dst, dst_off, dst_cap, out_len, n, known ? 1 : 0,
                                                    stream) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
    }
    void unwrap_from_host_at_async(const void* src, int64_t src_cap, const int64_t* src_off, void* dst, const int64_t* dst_off,
                                   const int32_t* dst_cap, int32_t* out_len, int32_t n, void* stream)
    {
        if (lz4b200_unwrap_batch_to_device_at_async(h_, src, src_cap, src_off, dst, dst_off, dst_cap, out_len, n, stream) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
    }
    // The same for an LZ4Stream (lz4b200_stream_encode_from_device_async, lz4b200_stream_decode_to_device_async): n bytes
    // of device memory as one stream in page-locked host memory, and back.  out_size is written by the device: the
    // stream's size, or the decoded size (LZ4B200_E_FORMAT when a chunk does not decode).  The decode walks the stream's
    // headers during the call, so src holds the whole stream when it is made.
    void stream_encode_to_host_async(const void* src, int64_t n, int32_t block_size, bool hc, void* dst, int64_t dst_cap,
                                     int64_t* out_size, void* stream)
    {
        if (lz4b200_stream_encode_from_device_async(h_, src, n, block_size, hc ? 1 : 0, dst, dst_cap, out_size, stream) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
    }
    void stream_decode_from_host_async(const void* src, int64_t n, void* dst, int64_t dst_cap, int64_t* out_size, void* stream)
    {
        if (lz4b200_stream_decode_to_device_async(h_, src, n, dst, dst_cap, out_size, stream) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
    }
    // The decode from the size the device wrote (lz4b200_stream_decode_to_device_at_async): src_size (device or page-locked
    // memory) is read and the headers are walked on the device, so the out_size of stream_encode_to_host_async above can be
    // passed straight in; only src_cap bytes of src are read, and block_size is the chunk size the stream was written with.
    void stream_decode_from_host_at_async(const void* src, int64_t src_cap, const int64_t* src_size, int32_t block_size, void* dst,
                                          int64_t dst_cap, int64_t* out_size, void* stream)
    {
        if (lz4b200_stream_decode_to_device_at_async(h_, src, src_cap, src_size, block_size, dst, dst_cap, out_size, stream) != LZ4B200_OK)
            throw std::runtime_error(lz4b200_last_error());
    }
private:
    lz4b200_ctx* h_ = nullptr;
};

class LZ4Codec {                                                         // static facade, src/LZ4/LZ4Codec.cs
public:
    static int MaximumOutputLength(int inputLength) { return inputLength + inputLength / 255 + 16; }   // :313-316
    static int Encode(const uint8_t* in, int io, int il, uint8_t* out, int oo, int ol) { return service().Encode(in, io, il, out, oo, ol); }
    static int EncodeHC(const uint8_t* in, int io, int il, uint8_t* out, int oo, int ol) { return service().EncodeHC(in, io, il, out, oo, ol); }
    static int Decode(const uint8_t* in, int io, int il, uint8_t* out, int oo, int ol, bool known = false) { return service().Decode(in, io, il, out, oo, ol, known); }

    static std::vector<uint8_t> Encode(const std::vector<uint8_t>& input) { return encode_vec(input, false); }       // :344-365
    static std::vector<uint8_t> EncodeHC(const std::vector<uint8_t>& input) { return encode_vec(input, true); }
    static std::vector<uint8_t> Decode(const std::vector<uint8_t>& input, int outputLength)                          // :448-462
    {
        if (input.empty()) return {};
        std::vector<uint8_t> out((size_t)outputLength);
        if (Decode(input.data(), 0, (int)input.size(), out.data(), 0, outputLength, true) != outputLength)
            throw std::invalid_argument("outputLength is not valid");
        return out;
    }
    static std::vector<uint8_t> Wrap(const std::vector<uint8_t>& in, Context& ctx) { return wrap(in, false, ctx); }  // :510-543
    static std::vector<uint8_t> WrapHC(const std::vector<uint8_t>& in, Context& ctx) { return wrap(in, true, ctx); }
    static std::vector<uint8_t> Unwrap(const std::vector<uint8_t>& in, Context& ctx)                                 // :574-599
    {
        const int size = lz4b200_unwrap_size(in.data(), (int)in.size());
        if (size < 0) throw std::invalid_argument("inputBuffer size is invalid or has been corrupted");
        std::vector<uint8_t> out((size_t)size + 1);
        const int r = lz4b200_unwrap(ctx.handle(), in.data(), (int)in.size(), out.data(), size);
        if (r < 0) throw std::invalid_argument("LZ4 block is corrupted, or invalid length has been given.");
        out.resize((size_t)r);
        return out;
    }
private:
    static ILZ4Service& service() { static CudaLZ4Service s; return s; }
    static std::vector<uint8_t> encode_vec(const std::vector<uint8_t>& input, bool hc)
    {
        if (input.empty()) return {};
        std::vector<uint8_t> out((size_t)MaximumOutputLength((int)input.size()));
        const int n = hc ? EncodeHC(input.data(), 0, (int)input.size(), out.data(), 0, (int)out.size())
                         : Encode(input.data(), 0, (int)input.size(), out.data(), 0, (int)out.size());
        if (n < 0) throw std::invalid_argument("Compression has been corrupted");
        out.resize((size_t)n);
        return out;
    }
    static std::vector<uint8_t> wrap(const std::vector<uint8_t>& in, bool hc, Context& ctx)
    {
        std::vector<uint8_t> out(in.size() + 8);
        const int r = lz4b200_wrap(ctx.handle(), in.data(), (int)in.size(), hc ? 1 : 0, out.data(), (int)out.size());
        if (r < 0) throw std::runtime_error(lz4b200_last_error());
        out.resize((size_t)r);
        return out;
    }
};

enum class LZ4StreamMode { Compress, Decompress };                       // src/LZ4/LZ4StreamMode.cs
enum LZ4StreamFlags { None = 0, InteractiveRead = 1, HighCompression = 2, IsolateInnerStream = 4, Default = 0 };   // LZ4StreamFlags.cs

// LZ4Stream over std::ostream / std::istream.  The wire format and the chunk boundaries are the reference's
// (src/LZ4/LZ4Stream.cs:239-312: a chunk per blockSize bytes written, a partial chunk on Flush/Close); the only
// difference is the dispatcher: up to `batchBlocks` buffered blocks go to the GPU in ONE batched call.
class LZ4Stream {
public:
    // maxBufferBytes caps the write buffer and the read-ahead (whole blocks / chunks); with InteractiveRead the reader hands
    // every chunk over as soon as it is read, like the reference (:376-401), instead of waiting for a batch of them.
    LZ4Stream(std::ostream& inner, Context& ctx, int flags = Default, int blockSize = 1024 * 1024, int batchBlocks = 256,
              size_t maxBufferBytes = 64u << 20)
        : out_(&inner), in_(nullptr), ctx_(ctx), hc_((flags & HighCompression) != 0), interactive_(false),
          blockSize_(std::max(16, blockSize)), batch_(std::max(1, batchBlocks)), maxBytes_(std::max<size_t>((size_t)blockSize_, maxBufferBytes)) {}
    LZ4Stream(std::istream& inner, Context& ctx, int flags = Default, int batchBlocks = 256, size_t maxBufferBytes = 64u << 20)
        : out_(nullptr), in_(&inner), ctx_(ctx), hc_(false), interactive_((flags & InteractiveRead) != 0),
          blockSize_(0), batch_(std::max(1, batchBlocks)), maxBytes_(std::max<size_t>(1, maxBufferBytes)) {}
    ~LZ4Stream() { try { Close(); } catch (...) {} }

    bool CanRead() const { return in_ != nullptr; }
    bool CanWrite() const { return out_ != nullptr; }
    bool CanSeek() const { return false; }

    void Write(const uint8_t* buffer, int offset, int count)             // :444-470
    {
        if (!CanWrite()) throw std::runtime_error("Operation 'Write' is not supported");
        pending_.insert(pending_.end(), buffer + offset, buffer + offset + count);
        const size_t full = std::min<size_t>((size_t)batch_, maxBytes_ / (size_t)blockSize_) * (size_t)blockSize_;
        // the reference flushes a full buffer only when MORE data arrives (:463-467); keep one byte back to do the same
        while (pending_.size() > full) emit(full);
    }
    void Flush() { if (CanWrite() && !pending_.empty()) emit(pending_.size()); }      // :337-340
    void Close() { if (!closed_) { Flush(); closed_ = true; } }

    int Read(uint8_t* buffer, int offset, int count)                     // :376-401
    {
        if (!CanRead()) throw std::runtime_error("Operation 'Read' is not supported");
        int total = 0;
        while (count > 0) {
            const int chunk = (int)std::min<size_t>((size_t)count, ready_.size() - rpos_);
            if (chunk > 0) {
                std::memcpy(buffer + offset, ready_.data() + rpos_, (size_t)chunk);
                rpos_ += (size_t)chunk; total += chunk;
                if (interactive_) break;
                offset += chunk; count -= chunk;
            } else if (!acquire()) break;
        }
        return total;
    }

private:
    void emit(size_t n)
    {
        const int64_t cap = lz4b200_stream_bound((int64_t)n, blockSize_);
        std::vector<uint8_t> buf((size_t)cap + 1);
        const int64_t w = lz4b200_stream_encode(ctx_.handle(), pending_.data(), (int64_t)n, blockSize_, hc_ ? 1 : 0, buf.data(), cap);
        if (w < 0) throw std::runtime_error(lz4b200_last_error());
        out_->write((const char*)buf.data(), (std::streamsize)w);
        pending_.erase(pending_.begin(), pending_.begin() + (std::ptrdiff_t)n);
    }
    // read up to batch_ chunks (headers walked like TryReadVarInt / AcquireNextChunk, :167-187,274-312), decode them together
    bool read_varint(uint64_t& v, bool first)
    {
        v = 0; int count = 0;
        for (;;) {
            const int c = in_->get();
            if (c == std::char_traits<char>::eof()) { if (first && count == 0) return false; throw std::runtime_error("Unexpected end of stream"); }
            raw_.push_back((uint8_t)c);
            v += (uint64_t)(c & 0x7F) << count; count += 7;
            if (!(c & 0x80) || count >= 64) return true;
        }
    }
    bool acquire()
    {
        raw_.clear(); ready_.clear(); rpos_ = 0;
        uint64_t decoded = 0;
        for (int k = 0; k < (interactive_ ? 1 : batch_) && decoded < maxBytes_; k++) {
            uint64_t flags, rawLen, compLen;
            if (!read_varint(flags, true)) break;
            read_varint(rawLen, false);
            compLen = rawLen;
            if (flags & 1) read_varint(compLen, false);
            // :288 corrupted; both lengths are ints in the reference -- nothing larger is ever resized to
            if (compLen > rawLen || rawLen > 0x7FFFFFFFull) throw std::runtime_error("Unexpected end of stream");
            decoded += rawLen;
            const size_t at = raw_.size();
            raw_.resize(at + (size_t)compLen);
            in_->read((char*)raw_.data() + at, (std::streamsize)compLen);
            if ((uint64_t)in_->gcount() != compLen) throw std::runtime_error("Unexpected end of stream");
        }
        if (raw_.empty()) return false;
        const int64_t total = lz4b200_stream_decoded_size(raw_.data(), (int64_t)raw_.size());
        if (total < 0) throw std::runtime_error("Unexpected end of stream");
        ready_.resize((size_t)total + 1);
        const int64_t r = lz4b200_stream_decode(ctx_.handle(), raw_.data(), (int64_t)raw_.size(), ready_.data(), total);
        if (r == LZ4B200_E_FORMAT) throw std::invalid_argument("LZ4 block is corrupted, or invalid length has been given.");
        if (r < 0) throw std::runtime_error(lz4b200_last_error());
        ready_.resize((size_t)total);
        return total > 0 || !raw_.empty();
    }

    std::ostream* out_; std::istream* in_; Context& ctx_;
    bool hc_, interactive_, closed_ = false;
    int blockSize_, batch_;
    size_t maxBytes_;
    std::vector<uint8_t> pending_, raw_, ready_;
    size_t rpos_ = 0;
};

}  // namespace LZ4
