// bazuka_b200 — one step of a precomputed hash plan: the per-node rule shared by the kernel (poseidon.cu,
// k_poseidon_plan_step) and the host compile of mpn_host.cu that the CPU test tier builds.
//
// A plan is a chain of steps; step k hashes n_k nodes of one arity (2, 4 or 5), and node j of the step hashes the operands
// ops[j * arity + 0 .. arity).  Each operand is tagged: with kPlanHost set, the low 31 bits index a value array the host
// uploaded with the plan (leaf scalars, clean siblings, defaults); without it, they index the outputs of step k - 1, which are
// still on the device.  So the structure of the work is fixed before any hash is known, and the whole plan runs as one launch
// per step with no host round trip in between (DESIGN.md §3.12).
#pragma once
#include "common.cuh"

namespace bzk {

constexpr uint32_t kPlanHost = 0x80000000u;

__host__ __device__ __forceinline__ const Fr *plan_operand(uint32_t op, const Fr *prev, const Fr *host) {
    return (op & kPlanHost) ? host + (op & ~kPlanHost) : prev + op;
}

// enqueue one step on the context's stream (poseidon.cu): d_ops[n][arity], d_prev = the previous step's outputs (device),
// d_host = the plan's value array (device), d_out[n]
int32_t poseidon_plan_step(bzk_ctx *ctx, uint32_t arity, const uint32_t *d_ops, size_t n, const Fr *d_prev, const Fr *d_host, Fr *d_out);

}  // namespace bzk
