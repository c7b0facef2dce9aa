// hd.h -- RB200_HD: a function compiled for the host and, under nvcc, for the device too (internal).  The container
// rules (container_format.h) and the decode-table formulas (tables.h) use it, so that the host parser and model build
// and the kernels of the async container decodes (container_decode.cuh) share one definition.
#pragma once

#ifdef __CUDACC__
#define RB200_HD __host__ __device__
#else
#define RB200_HD
#endif
