// conv2d.cuh -- parameter block shared by the SIMT and tensor-core NHWC conv2d kernels
#pragma once
struct Conv2dParams {
    const float* in; const float* w; const float* scale; const float* shift; float* out;
    int B, H, W, cin, in_cstride;
    int KH, KW, stride, pad;
    int Ho, Wo, cout;
    int OH, OW, os, oy0, ox0;        // physical output: pixel (ho*os+oy0, wo*os+ox0) of an (OH, OW) map
    int out_coff, out_cstride, relu;
    int tma_store;                   // tensor-core kernel: epilogue through shared memory + TMA stores (1: NHWC, 2: strided, os >= 2)
    const float* gshift; int gsize;  // optional per-row-group shift (linear layers only): + gshift[(row / gsize) * cout + n], row = y * W + x
    int grow0;                       // row index of pixel (0, 0) (tail calls of a linear layer)
    float* gmax; int gmax_rows;      // optional (linear layers): instead of storing y, atomically max-pool it over row groups of gmax_rows
                                     // (multiple of 128) into gmax[(row / gmax_rows) * cout + n] (pre-set to -inf): fused point-MLP + max-pool
};
