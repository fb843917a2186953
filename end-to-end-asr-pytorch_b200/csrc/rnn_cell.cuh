// The pointwise cell of the persistent recurrence kernels (csrc/lstm.cu, csrc/lstm_umma.cu): a compile-time parameter
// of every step kernel, so that a GRU layer runs on the LSTM's grid, planner, weight images and exchange protocols.
// Both cells see four gate slots per unit, gate-interleaved in `gates`, and one state value per unit in `cstate`:
//   LSTM  pre (i, f, g, o);  state register c;  stash (i, f, g, o) activated, cstate = c_t
//   GRU   pre (r, z, gi_n, gh_n) of the packed layout of ops.pack_decoder_weights("GRU"): slots 0 / 1 hold the input
//         and hidden products summed, slot 2 = x.W_in^T + b_in (its W_hh rows are zero), slot 3 = h.W_hn^T + b_hn (its
//         W_ih rows are zero);  state register h_{t-1};  stash (r, z, n, gh_n), cstate = h_t
// The backward reads the state of the previous step (c_{t-1} / h_{t-1}) through the same cstate indexing for both.
#pragma once
#include "common.cuh"

namespace b200asr {

enum RnnCell { CELL_LSTM = 0, CELL_GRU = 1 };

// Component q (0..3, a compile-time constant after inlining) of a float4.
__device__ __forceinline__ float f4_at(const float4& v, int q) {
    return q == 0 ? v.x : q == 1 ? v.y : q == 2 ? v.z : v.w;
}

// One forward step: pre(q) yields the pre-activation of slot q (evaluated in slot order, once each), s is the state
// register (c_{t-1} / h_{t-1}).  s becomes the value cstate keeps (c_t / h_t), g the activated-gate stash; cell_h
// then gives the output h_t.
template <int CELL, class Pre>
__device__ __forceinline__ void cell_fwd(const Pre& pre, float& s, float4& g) {
    if (CELL == CELL_LSTM) {
        const float ig = sigmoidf_(pre(0));
        const float fg = sigmoidf_(pre(1));
        const float gg = tanhf(pre(2));
        const float og = sigmoidf_(pre(3));
        s = fmaf(fg, s, ig * gg);
        g = make_float4(ig, fg, gg, og);
    } else {
        // ATen's GRUCell expression order (as csrc/gru.cu): n = tanh(gi_n + r * gh_n), h = (h_prev - n) * z + n, every
        // product and sum rounded on its own
        const float r = sigmoidf_(pre(0));
        const float z = sigmoidf_(pre(1));
        const float gin = pre(2);
        const float ghn = pre(3);
        const float n = tanhf(__fadd_rn(gin, __fmul_rn(ghn, r)));
        s = __fadd_rn(__fmul_rn(__fsub_rn(s, n), z), n);
        g = make_float4(r, z, n, ghn);
    }
}
// The output h_t of a step from cell_fwd's gates g and state s.
template <int CELL>
__device__ __forceinline__ float cell_h(const float4& g, float s) {
    return CELL == CELL_LSTM ? g.w * tanhf(s) : s;
}

// One backward step: the gate stash g, the state of this step st (c_t, LSTM only) and of the previous one sp
// (c_{t-1} / h_{t-1}, 0 at the first step), dh = dout + the recurrent partials, and the carry register of the later
// step (dc / dh.z) -> dg = d(loss)/d(pre-activation); carry becomes this step's.
template <int CELL>
__device__ __forceinline__ void cell_bwd(const float4& g, float st, float sp, float dh, float& carry, float4& dg) {
    if (CELL == CELL_LSTM) {
        const float ig = g.x, fg = g.y, gg = g.z, og = g.w;
        const float tc = tanhf(st);
        const float dc = carry + dh * og * (1.f - tc * tc);
        dg.x = dc * gg * ig * (1.f - ig);
        dg.y = dc * sp * fg * (1.f - fg);
        dg.z = dc * ig * (1.f - gg * gg);
        dg.w = dh * tc * og * (1.f - og);
        carry = dc * fg;
    } else {
        const float r = g.x, z = g.y, n = g.z, ghn = g.w;
        const float d = dh + carry;
        const float dgin = d * (1.f - z) * (1.f - n * n);
        dg.x = dgin * ghn * r * (1.f - r);
        dg.y = d * (sp - n) * z * (1.f - z);
        dg.z = dgin;
        dg.w = dgin * r;
        carry = d * z;
    }
}

}  // namespace b200asr
