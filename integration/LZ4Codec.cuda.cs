// LZ4Codec.cuda.cs -- the partial of LZ4.LZ4Codec that registers CudaLZ4Service, plus the batched entry points a GPU
// needs to be worth calling (one block per P/Invoke cannot feed it: INTEGRATION.md, "what to expect from one block").
//
// Shape of the change, following the reference's own per-platform partials (src/LZ4/LZ4Codec.windows.cs:66-94):
//   1. this file adds the service slot and its initializer;
//   2. the static constructor (src/LZ4/LZ4Codec.cs:76-101) gains one line:        Try(InitializeLZ4cuda);
//   3. SelectCodec (src/LZ4/LZ4Codec.cs:103-168) puts the slot in front where it pays: `_service_CUDA ??` ahead of
//      `_service_MM64` for encoderHC never (see INTEGRATION.md: LZ4HC stays on the CPU for single blocks), and for
//      encoder / decoder only when the application opted in (LZ4Codec.PreferCuda = true) -- a single 64 KiB block costs
//      a PCIe round trip, the CPU codecs win there; the batched calls below are where the GPU is ahead.
// Not compiled in this repository (no .NET toolchain in the build image).
using System;
using System.Runtime.CompilerServices;
using System.Runtime.InteropServices;
using LZ4.Services;

namespace LZ4
{
    public static partial class LZ4Codec
    {
        // ReSharper disable InconsistentNaming
        private static ILZ4Service _service_CUDA;

        /// <summary>Set before first use to rank the CUDA service ahead of the CPU services for single-block calls too.</summary>
        public static bool PreferCuda { get; set; }

        /// <summary>Initializes the codec backed by liblz4b200.</summary>
        [MethodImpl(MethodImplOptions.NoInlining)]
        private static void InitializeLZ4cuda()
        {
            _service_CUDA = TryService<CudaLZ4Service>();     // AutoTest()ed like every other service (src/LZ4/LZ4Codec.cs:173-239)
        }
        // ReSharper restore InconsistentNaming

        /// <summary>True when the batched entry points below are usable.</summary>
        public static bool CudaAvailable { get { return _service_CUDA != null; } }

        #region batched entry points (liblz4b200: include/lz4b200.h)

        private const string Library = "lz4b200";

        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern int lz4b200_create(out IntPtr ctx, int device);
        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern void lz4b200_destroy(IntPtr ctx);
        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern unsafe int lz4b200_encode_batch(IntPtr ctx, byte* src, long* srcOff, int* srcLen, byte* dst, long* dstOff,
                                                              int* dstCap, int* outLen, int nBlocks, int mode, int mem, IntPtr stream);
        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern unsafe int lz4b200_decode_batch(IntPtr ctx, byte* src, long* srcOff, int* srcLen, byte* dst, long* dstOff,
                                                              int* dstCap, int* outLen, int nBlocks, int knownLen, int mem, IntPtr stream);
        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern unsafe int lz4b200_measure_batch(IntPtr ctx, byte* src, long* srcOff, int* srcLen, int* dstCap, int* outLen,
                                                               int nBlocks, int knownLen, int mem, IntPtr stream);
        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern unsafe int lz4b200_decode_batch_packed(IntPtr ctx, byte* src, long* srcOff, int* srcLen, byte* dst,
                                                                     long dstTotalCap, long* outOff, int* outLen, int nBlocks, IntPtr stream);
        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern unsafe int lz4b200_decode_batch_packed_to_device(IntPtr ctx, byte* src, long* srcOff, int* srcLen, IntPtr dst,
                                                                               long dstTotalCap, long* outOff, int* outLen, int nBlocks, IntPtr stream);
        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern unsafe int lz4b200_wrap_batch(IntPtr ctx, byte* src, long* srcOff, int* srcLen, int highCompression,
                                                            byte* dst, long* dstOff, int* dstCap, int* outLen, int n);

        [ThreadStatic] private static IntPtr _cudaContext;        // one context per calling thread (contexts serialise their callers)

        private static IntPtr CudaContext()
        {
            if (_cudaContext == IntPtr.Zero && lz4b200_create(out _cudaContext, 0) != 0)
                throw new NotSupportedException("lz4b200: context creation failed");
            return _cudaContext;
        }

        /// <summary>Encodes blockCount blocks of blockSize bytes (the last one may be shorter) of <paramref name="input"/> in one
        /// GPU batch.  Block i's compressed bytes land in output at i * MaximumOutputLength(blockSize); lengths[i] is what
        /// <see cref="Encode(byte[],int,int,byte[],int,int)"/> would have returned for it (byte-identical output).</summary>
        public static unsafe void EncodeBlocks(byte[] input, int inputLength, int blockSize, byte[] output, int[] lengths, bool highCompression = false)
        {
            var n = (inputLength + blockSize - 1) / blockSize;
            var slot = MaximumOutputLength(blockSize);
            if (lengths.Length < n || output.Length < (long)n * slot) throw new ArgumentException("output buffers too small");
            var srcOff = new long[n]; var dstOff = new long[n]; var srcLen = new int[n]; var dstCap = new int[n];
            for (var i = 0; i < n; i++)
            {
                srcOff[i] = (long)i * blockSize; srcLen[i] = Math.Min(blockSize, inputLength - i * blockSize);
                dstOff[i] = (long)i * slot; dstCap[i] = slot;
            }
            fixed (byte* src = input) fixed (byte* dst = output) fixed (long* so = srcOff) fixed (long* dof = dstOff)
            fixed (int* sl = srcLen) fixed (int* dc = dstCap) fixed (int* ol = lengths)
            {
                var rc = lz4b200_encode_batch(CudaContext(), src, so, sl, dst, dof, dc, ol, n, highCompression ? 1 : 0, 0, IntPtr.Zero);
                if (rc != 0) throw new InvalidOperationException("lz4b200_encode_batch failed: " + rc);
            }
        }

        /// <summary>Decodes n blocks in one GPU batch: block i = input[inputOffsets[i], +inputLengths[i]) to
        /// output[i * blockSize, +outputLengths[i]) with known output lengths.  Throws like <see cref="Decode(byte[],int,int,byte[],int,int,bool)"/>
        /// when a block is corrupt.</summary>
        public static unsafe void DecodeBlocks(byte[] input, long[] inputOffsets, int[] inputLengths, byte[] output, int blockSize, int[] outputLengths)
        {
            var n = inputOffsets.Length;
            var dstOff = new long[n]; var consumed = new int[n];
            for (var i = 0; i < n; i++) dstOff[i] = (long)i * blockSize;
            fixed (byte* src = input) fixed (byte* dst = output) fixed (long* so = inputOffsets) fixed (long* dof = dstOff)
            fixed (int* sl = inputLengths) fixed (int* dc = outputLengths) fixed (int* ol = consumed)
            {
                var rc = lz4b200_decode_batch(CudaContext(), src, so, sl, dst, dof, dc, ol, n, 1, 0, IntPtr.Zero);
                if (rc != 0) throw new InvalidOperationException("lz4b200_decode_batch failed: " + rc);
            }
            for (var i = 0; i < n; i++)
                if (consumed[i] != inputLengths[i])
                    throw new ArgumentException("LZ4 block is corrupted, or invalid length has been given.");
        }

        /// <summary>The decoded size of each of n raw LZ4 blocks (input[inputOffsets[i], +inputLengths[i])) without decoding them:
        /// sizes[i] is what <see cref="Decode(byte[],int,int,byte[],int,int,bool)"/> with knownOutputLength = false and an
        /// unlimited output would return, or a negative value for a corrupt block.  Allocate, then decode with exact sizes.</summary>
        public static unsafe void MeasureBlocks(byte[] input, long[] inputOffsets, int[] inputLengths, int[] sizes)
        {
            var n = inputOffsets.Length;
            if (inputLengths.Length < n || sizes.Length < n) throw new ArgumentException("length arrays too small");
            fixed (byte* src = input) fixed (long* so = inputOffsets) fixed (int* sl = inputLengths) fixed (int* ol = sizes)
            {
                var rc = lz4b200_measure_batch(CudaContext(), src, so, sl, null, ol, n, 0, 0, IntPtr.Zero);
                if (rc != 0) throw new InvalidOperationException("lz4b200_measure_batch failed: " + rc);
            }
        }

        /// <summary>Decodes n raw LZ4 blocks whose decoded sizes nobody stored (input[inputOffsets[i], +inputLengths[i])) back to
        /// back into device memory of the context's GPU, in one pass over the compressed bytes.  offsets (n + 1 entries)
        /// receives where each block lies in <paramref name="deviceOutput"/> and, last, the total, which is returned;
        /// lengths[i] is what <see cref="Decode(byte[],int,int,byte[],int,int,bool)"/> with knownOutputLength = false would
        /// return, or a negative value for a corrupt block, which occupies no bytes.  When the total exceeds
        /// <paramref name="deviceCapacity"/> nothing of the output is valid (nothing is written outside it): allocate the
        /// returned total and call again.  Ordered behind the work already queued on <paramref name="stream"/>.</summary>
        public static unsafe long DecodeBlocksToDevice(byte[] input, long[] inputOffsets, int[] inputLengths, IntPtr deviceOutput,
                                                       long deviceCapacity, long[] offsets, int[] lengths, IntPtr stream = default(IntPtr))
        {
            var n = inputOffsets.Length;
            if (inputLengths.Length < n || lengths.Length < n || offsets.Length < n + 1) throw new ArgumentException("arrays too small");
            fixed (byte* src = input) fixed (long* so = inputOffsets) fixed (int* sl = inputLengths) fixed (long* oo = offsets)
            fixed (int* ol = lengths)
            {
                var rc = lz4b200_decode_batch_packed_to_device(CudaContext(), src, so, sl, deviceOutput, deviceCapacity, oo, ol, n, stream);
                if (rc != 0) throw new InvalidOperationException("lz4b200_decode_batch_packed_to_device failed: " + rc);
            }
            return offsets[n];
        }

        #endregion
    }
}
