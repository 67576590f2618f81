// The precision modes (PE_PREC_*, include/poseengine.h) in one table: the storage format of each mode and every per-mode rule
// of the host code.  Host code reads a mode's facts from its row; device code receives the storage format (PlaneFmt) and the
// element kinds as arguments and template parameters.  DESIGN.md section 3 explains the choices.
#pragma once
#include <cuda_runtime.h>   // __host__ __device__: device code uses PlaneFmt too

#include "../../include/poseengine.h"

namespace pe {

// Element kind of a storage plane.  Facts that depend on the kind alone are functions of it.
// ELEM_U8: the non-negative activations of PE_PREC_S8X1 | PE_PREC_FLAG_U8 (plan.cpp), read as u8 against s8 weights.
enum PlaneElem { ELEM_BF16 = 0, ELEM_F16 = 1, ELEM_E4M3 = 2, ELEM_S8 = 3, ELEM_U8 = 4 };
constexpr int NUM_ELEMS = 5;
__host__ __device__ constexpr int elem_size(PlaneElem e) { return e == ELEM_E4M3 || e == ELEM_S8 || e == ELEM_U8 ? 1 : 2; }   // bytes
// pack_conv_weights scales a layer's weights by a power of two so that max|w| lies in [2^(top-1), 2^top): fp16 [2^13, 2^14) keeps
// the lo plane of small weights out of the subnormals, e4m3 [128, 256) stays below the largest finite 448 and keeps weights down to
// max|w| * 2^-13 normal.  0: no scaling (bf16 has fp32's range; s8 scales each output channel, s8.h).  A fact of the element kind,
// not of the mode: E4M3X1 packs conv1_1's weights in fp16.
constexpr int weight_top(PlaneElem e) { return e == ELEM_F16 ? 14 : e == ELEM_E4M3 ? 8 : 0; }

// Storage of activations and packed weights: `planes` planes of kind `elem` whose sum is the value; 0 planes: fp32.
struct PlaneFmt {
    int planes; PlaneElem elem;
    __host__ __device__ bool f16() const { return elem == ELEM_F16; }
    __host__ __device__ bool e4m3() const { return elem == ELEM_E4M3; }
    __host__ __device__ bool s8() const { return elem == ELEM_S8; }
    __host__ __device__ bool u8() const { return elem == ELEM_U8; }
    __host__ __device__ int elem_bytes() const { return planes == 0 ? 4 : elem_size(elem); }
};

struct Precision {
    PlaneFmt fmt;                  // activations and packed weights
    PlaneElem input_elem;          // the im2col'ed net input, one plane, and so conv1_1's packed weights
    int act_cpad;                  // channel granularity of every activation: one K block of the conv kernel (common.h)
    int kp_input;                  // channel pitch of the im2col'ed net input (27 values)
    int slot_align;                // Concat slots start at multiples of this many channels: 16 bytes of the element (plan.cpp)
    bool chunked;                  // hi*hi accumulates in chunks summed with round-to-nearest (conv_tc.cu); else one chain over K
    int range_top;                 // pe_calibrate puts every stored maximum into [2^(range_top-1), 2^range_top); 0: no range scales
    float range_limit;             // pe_range_status: PE_ERR_RANGE when a layer's largest stored value reaches this ...
    float range_floor;             // ... or stays below this
    const char* range_floor_text;  // the floor and the planes as pe_range_status's messages name them
    const char* range_what;
    float net_input_scale;         // stored net input = true value x this
    bool needs_calibration;        // a forward before pe_calibrate is PE_ERR_STATE
    long long max_k;               // largest K = taps x padded input channels of a layer; 0: no bound
    bool per_channel_epilogue;     // one epilogue factor per output channel after the biases in the packed buffer; else one per layer
    bool ranged() const { return range_top != 0; }   // range scales and range tracking
};

// Row i describes PE_PREC_* = i.
//   E4M3X1 keeps the net input in fp16: p/256 - 0.5 is exact there, not in e4m3.
//   S8X1 stores the net input as p - 128 = (p/256 - 0.5) x 2^8.  Its sums are exact, so nothing is chunked, and
//   |acc| <= 128 x 127 x K stays inside s32 up to K = 132104.
//   Calibration targets: fp16 [32, 64), 1000x below 65504; e4m3 [64, 128), 3.5-7x below 448 with values down to max x 2^-12
//   still normal; s8 [32, 64): 6 bits and 2-4x headroom for frames busier than the calibration frame.
//   Range floors: fp16 2^-10 (below it the lo plane lives in subnormals); e4m3 2^-2, 16x above the smallest normal, so that
//   values a sixteenth of the maximum stay normal; s8 4 (under 3 bits).
inline constexpr Precision PRECISIONS[] = {
    // fmt, input_elem, act_cpad, kp_input, slot_align, chunked, range_top, range_limit, range_floor, range_floor_text, range_what,
    // net_input_scale, needs_calibration, max_k, per_channel_epilogue
    {{0, ELEM_BF16}, ELEM_BF16, 16, 32, 8, false, 0, 0.f, 0.f, nullptr, nullptr, 1.f, false, 0, false},                              // FP32_SIMT
    {{1, ELEM_BF16}, ELEM_BF16, 64, 64, 8, false, 0, 0.f, 0.f, nullptr, nullptr, 1.f, false, 0, false},                              // BF16X1
    {{2, ELEM_F16}, ELEM_F16, 64, 64, 8, true, 6, 65504.f, 9.765625e-4f, "2^-10", "the fp16 planes", 1.f, false, 0, false},          // F16X2
    {{3, ELEM_BF16}, ELEM_BF16, 64, 64, 8, true, 0, 0.f, 0.f, nullptr, nullptr, 1.f, false, 0, false},                               // BF16X3
    {{1, ELEM_F16}, ELEM_F16, 64, 64, 8, true, 6, 65504.f, 9.765625e-4f, "2^-10", "the fp16 planes", 1.f, false, 0, false},          // F16X1
    {{1, ELEM_E4M3}, ELEM_F16, 128, 64, 16, true, 7, 448.f, 0.25f, "2^-2", "the e4m3 planes", 1.f, false, 0, false},                 // E4M3X1
    {{1, ELEM_S8}, ELEM_S8, 128, 128, 16, false, 6, 127.f, 4.f, "4", "the s8 planes", 256.f, true, 132104, true},                    // S8X1
};
constexpr int NUM_PRECISIONS = sizeof PRECISIONS / sizeof PRECISIONS[0];
static_assert(NUM_PRECISIONS == PE_PREC_S8X1 + 1, "one row per PE_PREC_* mode up to S8X1");

// PE_PREC_S8X2, the 16-bit integer mode: v in [-32768, 32639] stored as two s8 planes, hi = (v + 128) >> 8 and lo = v - 256 hi
// (s8.h), hi*hi into one s32 accumulator and hi*lo + lo*hi into a second, both over the whole K (exact, so nothing is
// chunked); lo*lo is dropped.  |acc_c| <= (128 x 128 + 128 x 127) x K stays inside s32 up to K = 65793.  The net input keeps
// S8X1's im2col bytes in the hi plane with a zero lo plane, so it stores (p - 128) x 2^8 = (p/256 - 0.5) x 2^16.
// Calibration target [2^13, 2^14): the 2-4x headroom of S8X1's [32, 64) below the largest stored value 32639.  Range floor
// 2^8: below it the hi plane carries nothing and the layer runs on the lo plane's 8 bits.  Its own row after PRECISIONS,
// which holds the modes up to S8X1; precision() answers for every mode.
inline constexpr Precision S8X2_ROW =
    {{2, ELEM_S8}, ELEM_S8, 128, 128, 16, false, 14, 32639.f, 256.f, "2^8", "the s8 plane pairs", 65536.f, true, 65793, true};
static_assert((128LL * 128 + 128LL * 127) * 65793 <= 2147483647LL && (128LL * 128 + 128LL * 127) * 65794 > 2147483647LL,
              "65793: the largest K of an S8X2 layer");
// The PE_PREC_* values with a row: 0 .. PE_PREC_S8X1 and PE_PREC_S8X2 (8; 7 is not assigned, poseengine.h)
constexpr bool known_mode(int pe_prec) { return (pe_prec >= 0 && pe_prec < NUM_PRECISIONS) || pe_prec == PE_PREC_S8X2; }
inline const Precision& precision(int pe_prec) { return pe_prec == PE_PREC_S8X2 ? S8X2_ROW : PRECISIONS[pe_prec]; }   // known_mode(pe_prec)

// The u8 activations of PE_PREC_S8X1 | PE_PREC_FLAG_U8 (plan.cpp: post-ReLU values read only by integer layers), outside
// PRECISIONS since they are no mode of their own.  S8X1's layout and per-channel epilogue; u8 x s8 sums, |acc| <= 255 x 127 x K,
// stay inside s32 up to K = 66311.  Calibration target [64, 128): the sign bit s8 spends on these values goes to one more bit
// of magnitude, with the 2-4x headroom of S8X1's [32, 64).  Range limit 255, floor 8 (under 3 bits, as S8X1's 4).
inline constexpr Precision U8_ACTIVATIONS =
    {{1, ELEM_U8}, ELEM_S8, 128, 128, 16, false, 7, 255.f, 8.f, "8", "the u8 planes", 256.f, true, 66311, true};
static_assert(255LL * 127 * 66311 <= 2147483647LL && 255LL * 127 * 66312 > 2147483647LL, "66311: the largest K of a u8 layer");

// The row of a layer or activation of element kind k in an engine of mode `base`.  The one-plane 16-bit and 8-bit modes give
// each kind one row - fp16: F16X1, e4m3: E4M3X1, s8: S8X1, u8: U8_ACTIVATIONS - so that a layer of another kind than the mode's
// (E4M3X1's fp16 net input, the fp16 layers of pe_create_mixed, the u8 layers of PE_PREC_FLAG_U8) follows its own kind's
// arithmetic, pads and range.  Other modes: their own row.
inline const Precision& elem_row(const Precision& base, PlaneElem k) {
    if (k == ELEM_U8) return U8_ACTIVATIONS;
    if (base.fmt.planes != 1 || k == ELEM_BF16) return base;
    return precision(k == ELEM_F16 ? PE_PREC_F16X1 : k == ELEM_E4M3 ? PE_PREC_E4M3X1 : PE_PREC_S8X1);
}

}  // namespace pe
