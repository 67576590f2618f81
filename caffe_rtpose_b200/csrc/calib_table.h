// Calibration tables (pe_calibration_get / pe_calibration_set, include/poseengine.h): the per-layer power-of-two range scales of an
// engine as text, one fact per line, so that a person can read and diff it:
//   pe_calibration 1
//   precision 6
//   weights 9f3a0c1e5b7d2468      FNV-1a 64 of every conv layer's name, fp32 weights and biases, in plan order
//   layer conv1_1 s8 -3           every conv layer that stores an activation, in plan order: name, stored kind, log2 scale
// '#' starts a comment that runs to the end of the line.  Host code only (no CUDA), so that a fuzzer can build it on its own.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <string>
#include <vector>

namespace pe {

constexpr int CALIB_TABLE_VERSION = 1;
constexpr int CALIB_MAX_LOG2 = 100;   // pe_calibrate clamps every exponent to [-100, 100]

struct CalibLayer { std::string name, kind; int log2_scale = 0; };
struct CalibTable { int precision = 0; uint64_t weights = 0; std::vector<CalibLayer> layers; };

struct Fnv1a64 {
    uint64_t h = 1469598103934665603ull;
    void add(const void* p, size_t n) {
        const unsigned char* b = (const unsigned char*)p;
        for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 1099511628211ull; }
    }
};

std::string write_calibration_table(const CalibTable& t);

// Reads `text` and checks it against the engine's own table `expect` (its precision, weights hash, layer names and kinds; the
// exponents of `expect` are not read).  On success log2_out[j] is the exponent of expect.layers[j].  Otherwise -1, and err names
// the line or the layer.
int read_calibration_table(const char* text, const CalibTable& expect, std::vector<int>& log2_out, std::string& err);

}  // namespace pe
