/*
 * NativePca -- JNI binding of ONE vpca_ctx of libvpca.so (include/vpca.h), 1:1 with the C ABI.  A driver that uses
 * all GPUs of its host holds a NativePcaPool (NativePcaPool.scala) instead; this class is the single-GPU form and the
 * home of the pinned-buffer helpers.
 *
 * No JVM, scalac or jni.h in this repository's image (SURVEY.md 8c): this file is source for the maintainer of
 * googlegenomics/spark-examples.  Its native half, vpca_jni.c, IS compiled and executed here -- against a stub jni.h
 * and a mock JNIEnv (tests/jni_harness.c); spark_examples_b200/native.py is the same binding over ctypes.
 */
package com.google.cloud.genomics.spark.examples

import java.nio.ByteBuffer

object NativePca {
  System.loadLibrary("vpca_jni") // links against libvpca.so

  val DTYPE_I8 = 0
  val DTYPE_BF16 = 1
  val DTYPE_E2M1 = 2 // packed 4-bit cells (expanded to int8 on the device; exact for 0/1/2)

  // every native method throws on a negative vpca_status: IndexOutOfBoundsException for a sample index outside [0, N)
  // (what Breeze throws at VariantsPca.scala:188), IllegalArgumentException, OutOfMemoryError, else RuntimeException
  @native def create(nSamples: Int, device: Int, dtype: Int, numPc: Int, maxMultiplicity: Int,
                     partitionsInFlight: Int): Long
  @native def destroy(handle: Long): Unit
  @native def reset(handle: Long): Unit
  /** offsets: nv + 1 entries; sampleIdx: the concatenated rows of one batch of RDD[Seq[Int]] (VariantsPca.scala:153-168). */
  @native def accumulateCalls(handle: Long, partitionId: Long, offsets: Array[Long], sampleIdx: Array[Int], nv: Long): Unit
  /** Same rows with 16-bit sample indices (N <= 65536): half the PCIe bytes. */
  @native def accumulateCallsU16(handle: Long, partitionId: Long, offsets: Array[Long], sampleIdx: Array[Short], nv: Long): Unit
  /** Same rows packed by the task straight into pinned direct buffers (allocPinned; little-endian longs / ints or
   *  shorts): no copy on the host, the copy engines read the buffers at full PCIe rate. */
  @native def accumulateCallsDirect(handle: Long, partitionId: Long, offsets: ByteBuffer, sampleIdx: ByteBuffer, nv: Long,
                                    idxBytes: Int): Unit
  /** One N-bit bitmap per variant, bit s (LSB first) = hasVariation of sample s; rows strideBytes apart. */
  @native def accumulateBits(handle: Long, partitionId: Long, bits: Array[Byte], nv: Long, strideBytes: Long): Unit
  /** PLINK .bed rows as on disk (2 bits per sample); countedAllele 1 = A1, 2 = A2. */
  @native def accumulateBed(handle: Long, partitionId: Long, rows: Array[Byte], nv: Long, strideBytes: Long,
                            countedAllele: Int): Unit
  /** joinDatasets (mode 0, VariantsPca.scala:115-128) / mergeDatasets (mode 1, :136-148) on the GPU: rows of all datasets
   *  (dataset 0 first; the calls with variation as callset indices) and the bytes getVariantKey (:65-73) would hash, per
   *  row.  The joined rows stay on the device; returns their number.  Follow with accumulateJoined + commit. */
  @native def joinRows(handle: Long, mode: Int, variantSetCount: Int, nLeft: Long, keyBytes: Array[Byte],
                       keyOffsets: Array[Long], offsets: Array[Long], sampleIdx: Array[Int], nRows: Long): Long
  /** The joined rows as a CSR pair (offsets: rows + 1 entries, sampleIdx: at least the number of calls). */
  @native def joinFetch(handle: Long, outOffsets: Array[Long], outSampleIdx: Array[Int]): Unit
  /** Rows / calls of the retained join. */
  @native def joinRowCount(handle: Long): Long
  @native def joinCallCount(handle: Long): Long
  @native def accumulateJoined(handle: Long, partitionId: Long): Unit
  @native def commit(handle: Long, partitionId: Long): Unit
  @native def abort(handle: Long, partitionId: Long): Unit
  @native def finalizeGram(handle: Long): Unit
  /** Row-major N x N (the collected RDD[((Int, Int), Int)] of VariantsPca.scala:182-191 in key order). */
  @native def getGram(handle: Long, nSamples: Int, out: Array[Int]): Unit
  @native def setGram(handle: Long, nSamples: Int, gram: Array[Int]): Unit
  @native def gramDevicePtr(handle: Long): Long
  /** vecs: N x k column-major -- the layout of `pca.toArray` (VariantsPca.scala:227); returns nonZeroRows (:207). */
  @native def computePca(handle: Long, nSamples: Int, k: Int, vecs: Array[Double], evals: Array[Double]): Int

  /** Page-locked host memory as a direct ByteBuffer (set order(ByteOrder.LITTLE_ENDIAN) before writing). */
  @native def allocPinned(bytes: Long): ByteBuffer
  @native def freePinned(buffer: ByteBuffer): Unit
}
