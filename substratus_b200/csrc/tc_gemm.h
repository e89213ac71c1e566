// tc_gemm.h — launch API of the wgmma/TMA projection kernel and the prefill RMSNorm.
#pragma once
#include "kernels.h"

struct alignas(64) TcTensorMap {
  unsigned char bytes[128];  // CUtensorMap (opaque, 64-byte aligned)
};

// 2-D K-major bf16 tensor map over global [rows, cols] (row pitch ld elements); TMA box = [box_rows, 64], 128B swizzle
cudaError_t tc_make_tmap(TcTensorMap* out, const bf16* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows);
int tc_pick_tn(int M);          // token-tile width (wgmma N) for M token rows: 16 | 32 | 64 | 128
int tc_pick_tn_prefill(int M, int N, int n_sm);  // per projection [N out rows]: 128 | 256 above 128 token rows (waves x tile cost)
int tc_weight_box_rows();       // 128
// Y = X * W^T with the fused epilogue `epi` (GemvEpi); tmA = weights (box 128 rows), tmB = activations (box tn rows)
cudaError_t launch_tc_gemm(const TcTensorMap& tmA, const TcTensorMap& tmB, int tn, const GemvArgs& a, int epi, const LaunchCfg& lc);
cudaError_t launch_rmsnorm(const bf16* x, const bf16* w, bf16* out, int M, int K, float eps, const LaunchCfg& lc);
cudaError_t launch_layernorm(const bf16* x, const bf16* w, const bf16* b, bf16* out, int M, int K, float eps, const LaunchCfg& lc);
// The stream-K decode kernel takes its fp32 partial-tile workspace from LaunchCfg (sk_part = sk_slots * 64 * 128 floats,
// sk_flags = sk_slots zeroed words, sk_slots >= 2 * SM count); without one launch_tc_gemm uses one CTA per 128-row tile.
