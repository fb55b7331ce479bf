// Limb formats of the two-limb mode (UDH_NUMERIC_BF16X3): forward operands (activations, forward weights, fc1's weight
// mirror) and backward operands (gradients, mirrored conv weights).
// wgmma multiplies operands of one format, so both operands of every MMA share a limb format.  fp16 limbs would carry 22
// bits instead of 16, but the weight gradient multiplies activations with gradients, and gradients (1e-8 .. 1e-2) do not
// fit fp16's range without per-tensor loss scaling; bf16 limbs need no scaling anywhere, so every stream uses them.
#pragma once
#include "tc_common.cuh"

namespace udh {
constexpr int kX3Fwd = tc::kFmtBF16;
constexpr int kX3Grad = tc::kFmtBF16;
}  // namespace udh
