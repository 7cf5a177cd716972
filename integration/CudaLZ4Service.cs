// CudaLZ4Service.cs -- ILZ4Service over liblz4b200 (the H100 / sm_90a LZ4 block codec of this repository).
//
// Drop into src/LZ4/Services/ of lz4net next to CppMM64LZ4Service.cs (which this file mirrors in shape:
// src/LZ4/Services/CppMM64LZ4Service.cs:38-51) and compile it into the LZ4 assembly -- ILZ4Service is internal
// (src/LZ4/ILZ4Service.cs:30-36).  The managed side only pins the arrays and applies the C# boundary conventions that
// lz4net's own wrappers apply around the C code (src/LZ4ps/LZ4Codec.Safe.cs:392-415,522-551,707-724):
//   * empty input -> 0 without calling the codec            (src/LZ4ps/LZ4Codec.cs:156-160)
//   * EncodeHC failure (C returns 0) -> -1                   (src/LZ4ps/LZ4Codec.Safe.cs:721-723)
//   * known-size decode that does not consume exactly inputLength bytes, or any negative result -> ArgumentException
//                                                            (src/LZ4ps/LZ4Codec.Safe.cs:539-549)
// The entry points are the four functions LZ4mm / LZ4cc call (src/LZ4cc/LZ4Codec.64.cpp:35,88,95,143), exported by
// liblz4b200 under the lz4b200_ prefix (include/lz4b200.h); lz4b200_uncompress takes the compressed length as an extra
// argument because the bytes are staged to the device.
//
// Not compiled in this repository (no .NET toolchain in the build image); INTEGRATION.md lists the three lines that hook
// it into LZ4Codec's static constructor and SelectCodec.
using System;
using System.Runtime.InteropServices;

namespace LZ4.Services
{
    // ReSharper disable once InconsistentNaming
    internal unsafe class CudaLZ4Service : ILZ4Service
    {
        private const string Library = "lz4b200";   // liblz4b200.so / lz4b200.dll on the loader path

        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern int lz4b200_device_count();

        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern int lz4b200_compress_limitedOutput(byte* source, byte* dest, int isize, int maxOutputSize);

        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern int lz4b200_compressHC_limitedOutput(byte* source, byte* dest, int isize, int maxOutputSize);

        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern int lz4b200_uncompress(byte* source, byte* dest, int isize, int osize);

        [DllImport(Library, CallingConvention = CallingConvention.Cdecl)]
        private static extern int lz4b200_uncompress_unknownOutputSize(byte* source, byte* dest, int isize, int maxOutputSize);

        /// <summary>Throws unless a compute-capability 9.x device is usable: TryService() then discards this service,
        /// exactly like a native service whose assembly fails to load (src/LZ4/LZ4Codec.cs:278-290).</summary>
        public CudaLZ4Service()
        {
            if (lz4b200_device_count() < 1)
                throw new NotSupportedException("lz4b200: no sm_90 device");
        }

        public string CodecName
        {
            get { return "CUDA H100"; }
        }

        // the argument rules of src/LZ4ps/LZ4Codec.cs:151-170 (negative length = to the end of the array)
        private static void Check(byte[] input, int inputOffset, ref int inputLength, byte[] output, int outputOffset, ref int outputLength)
        {
            if (inputLength < 0) inputLength = input.Length - inputOffset;
            if (inputLength == 0) { outputLength = 0; return; }
            if (input == null) throw new ArgumentNullException("input");
            if ((uint)inputOffset > (uint)input.Length - (uint)inputLength) throw new ArgumentException("inputOffset and inputLength are invalid for given input");
            if (outputLength < 0) outputLength = output.Length - outputOffset;
            if (output == null) throw new ArgumentNullException("output");
            if ((uint)outputOffset > (uint)output.Length - (uint)outputLength) throw new ArgumentException("outputOffset and outputLength are invalid for given output");
        }

        public int Encode(byte[] input, int inputOffset, int inputLength, byte[] output, int outputOffset, int outputLength)
        {
            Check(input, inputOffset, ref inputLength, output, outputOffset, ref outputLength);
            if (outputLength == 0) return 0;
            fixed (byte* src = &input[inputOffset])
            fixed (byte* dst = &output[outputOffset])
                return lz4b200_compress_limitedOutput(src, dst, inputLength, outputLength);
        }

        public int EncodeHC(byte[] input, int inputOffset, int inputLength, byte[] output, int outputOffset, int outputLength)
        {
            if (inputLength == 0) return 0;
            Check(input, inputOffset, ref inputLength, output, outputOffset, ref outputLength);
            if (outputLength == 0) return -1;
            fixed (byte* src = &input[inputOffset])
            fixed (byte* dst = &output[outputOffset])
            {
                var length = lz4b200_compressHC_limitedOutput(src, dst, inputLength, outputLength);
                return length <= 0 ? -1 : length;
            }
        }

        public int Decode(byte[] input, int inputOffset, int inputLength, byte[] output, int outputOffset, int outputLength, bool knownOutputLength)
        {
            Check(input, inputOffset, ref inputLength, output, outputOffset, ref outputLength);
            if (outputLength == 0) return 0;
            fixed (byte* src = &input[inputOffset])
            fixed (byte* dst = &output[outputOffset])
            {
                if (knownOutputLength)
                {
                    var read = lz4b200_uncompress(src, dst, inputLength, outputLength);
                    if (read != inputLength)
                        throw new ArgumentException("LZ4 block is corrupted, or invalid length has been given.");
                    return outputLength;
                }
                var written = lz4b200_uncompress_unknownOutputSize(src, dst, inputLength, outputLength);
                if (written < 0)
                    throw new ArgumentException("LZ4 block is corrupted, or invalid length has been given.");
                return written;
            }
        }
    }
}
