// Checks and mutation fuzzer for the calibration table reader (csrc/calib_table.cpp): a table is a user file (--calibration_table).
// Built with -fsanitize=address,undefined by tests/test_calibration_table.py; any finding aborts.
// usage: fuzz_calibration_table cases              one line per named refusal: "<case> <rc> <message>"
//        fuzz_calibration_table fuzz <iterations>  mutations of valid tables: every outcome is a table or a message, never a crash
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "calib_table.h"

using pe::CalibTable;

static CalibTable engine_table(int layers, int precision, const char* kind) {
    CalibTable t;
    t.precision = precision;
    pe::Fnv1a64 h;
    h.add("weights", 7);
    t.weights = h.h;
    for (int i = 0; i < layers; i++) t.layers.push_back({"conv" + std::to_string(i + 1) + "_1", (i < 2 ? "f16" : kind), (i * 7) % 23 - 11});
    return t;
}

static int check(const std::string& text, const CalibTable& want, std::string& err) {
    std::vector<int> k;
    const int rc = pe::read_calibration_table(text.c_str(), want, k, err);
    if (rc == 0) {
        if (k.size() != want.layers.size()) { printf("accepted with %zu exponents for %zu layers\n", k.size(), want.layers.size()); exit(3); }
        for (int v : k) if (v < -pe::CALIB_MAX_LOG2 || v > pe::CALIB_MAX_LOG2) { printf("accepted exponent %d\n", v); exit(3); }
    } else if (err.empty()) {
        printf("refused without a message\n");
        exit(3);
    }
    return rc;
}

static std::string replace(std::string s, const std::string& a, const std::string& b) {
    const size_t p = s.find(a);
    if (p == std::string::npos) { printf("case text '%s' not found\n", a.c_str()); exit(4); }
    return s.replace(p, a.size(), b);
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    const CalibTable want = engine_table(6, 6, "s8");
    const std::string good = pe::write_calibration_table(want);
    if (!strcmp(argv[1], "cases")) {
        const std::string w = want.layers[2].name + " s8 " + std::to_string(want.layers[2].log2_scale);
        char hash[17];
        snprintf(hash, sizeof hash, "%016llx", (unsigned long long)want.weights);
        const std::string l2 = "layer " + want.layers[2].name + " s8 " + std::to_string(want.layers[2].log2_scale) + "\n";
        const std::string l3 = "layer " + want.layers[3].name + " s8 " + std::to_string(want.layers[3].log2_scale) + "\n";
        const std::vector<std::pair<std::string, std::string>> cases = {
            {"valid", good},
            {"valid_comments", "# saved by hand\n" + replace(good, "\nprecision 6\n", "\nprecision 6   # INT8\n\n")},
            {"empty", ""},
            {"version", replace(good, "pe_calibration 1", "pe_calibration 2")},
            {"precision", replace(good, "precision 6", "precision 5")},
            {"weights", replace(good, hash, "0000000000000000")},
            {"weights_syntax", replace(good, hash, "12345")},
            {"missing", replace(good, l2, "")},
            {"missing_last", good.substr(0, good.rfind("layer "))},
            {"duplicated", replace(good, l2, l2 + l2)},
            {"out_of_order", replace(good, l2 + l3, l3 + l2)},
            {"unknown", replace(good, l2, "layer conv9_9 s8 0\n")},
            {"kind", replace(good, w, want.layers[2].name + " f16 " + std::to_string(want.layers[2].log2_scale))},
            {"exponent", replace(good, w, want.layers[2].name + " s8 101")},
            {"exponent_syntax", replace(good, w, want.layers[2].name + " s8 3.5")},
            {"trailing_text", replace(good, w, w + " extra")},
            {"trailing_line", good + "end\n"},
            {"header_order", replace(good, "precision 6\n", "") + "precision 6\n"},
        };
        for (const auto& c : cases) {
            std::string err;
            const int rc = check(c.second, want, err);
            printf("%s %d %s\n", c.first.c_str(), rc, rc ? err.c_str() : "ok");
        }
        return 0;
    }
    if (strcmp(argv[1], "fuzz") || argc < 3) return 2;
    const int iters = atoi(argv[2]);
    uint64_t s = 7654321;
    auto rnd = [&]() { s = s * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(s >> 33); };
    static const char* const kTokens[] = {" ", "\n", "#", "layer ", "precision ", "weights ", "pe_calibration ", "-", "+", "0", "101", "-100",
                                          "2147483648", "99999999999999999999", "ffffffffffffffff", "s8", "f16", "e4m3", "\t", "\r", "conv1_1"};
    long accepted = 0, rejected = 0;
    const std::vector<CalibTable> seeds = {want, engine_table(1, 5, "e4m3"), engine_table(40, 2, "f16")};
    for (int it = 0; it < iters; it++) {
        const CalibTable& t = seeds[it % seeds.size()];
        std::string d = pe::write_calibration_table(t);
        const int nm = 1 + rnd() % 4;
        for (int k = 0; k < nm && !d.empty(); k++) {
            const int kind = rnd() % 6;
            const size_t p = rnd() % d.size();
            if (kind == 0) d[p] = (char)rnd();
            else if (kind == 1) d.resize(p);
            else if (kind == 2) d.insert(p, kTokens[rnd() % (sizeof kTokens / sizeof *kTokens)]);
            else if (kind == 3) { const size_t e = d.find('\n', p); d.erase(p, e == std::string::npos ? std::string::npos : e - p + 1); }
            else if (kind == 4) { const size_t b = d.rfind('\n', p); const size_t e = d.find('\n', p); if (e != std::string::npos) d.insert(e + 1, d.substr(b == std::string::npos ? 0 : b + 1, e - (b == std::string::npos ? 0 : b + 1)) + "\n"); }
            else { const size_t q = d.find_first_of("0123456789", p); if (q != std::string::npos) d[q] = (char)('0' + rnd() % 10); }
        }
        std::string err;
        if (check(d, t, err) == 0) accepted++; else rejected++;
    }
    printf("accepted %ld rejected %ld\n", accepted, rejected);
    return 0;
}
