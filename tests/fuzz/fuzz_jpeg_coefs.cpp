// Mutation fuzzer for the JPEG coefficient stage (pe_jpeg_read_coefs) and the host reconstruction of its output
// (pe_jpeg_coefs_to_bgr).  Built with -fsanitize=address,undefined by tests/test_jpeg_coefs.py; any finding aborts.  Besides memory
// safety it checks, on every mutated stream, that the coefficient stage accepts and rejects exactly what pe_decode_jpeg does and that
// the reconstruction of accepted streams gives pe_decode_jpeg's pixels.
// usage: fuzz_jpeg_coefs <iterations> <file.jpg>...
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "poseengine.h"

static std::vector<uint8_t> slurp(const char* p) {
    std::vector<uint8_t> d;
    FILE* f = fopen(p, "rb");
    if (!f) return d;
    fseek(f, 0, SEEK_END);
    const long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    d.resize(n > 0 ? (size_t)n : 0);
    if (fread(d.data(), 1, d.size(), f) != d.size()) d.clear();
    fclose(f);
    return d;
}

// one stream: 0 = same outcome on both paths, 1 = mismatch (printed)
static int check(const std::vector<uint8_t>& d, long& ok, long& rejected) {
    const long long n = pe_jpeg_read_coefs(d.data(), (long long)d.size(), nullptr, 0);
    int w = 0, h = 0;
    const int rc0 = pe_decode_jpeg(d.data(), (long long)d.size(), &w, &h, nullptr, 0);
    if ((n > 0) != (rc0 == 0) || (n < 0 && n != rc0)) { printf("size query: coefs %lld, decode %d\n", n, rc0); return 1; }
    if (n <= 0 || (long long)w * h > 4000000 || n > 64000000) { rejected++; return 0; }
    std::vector<uint8_t> ref((size_t)w * h * 3), got((size_t)w * h * 3);   // exact sizes: ASAN sees any write past them
    std::vector<uint8_t> buf((size_t)n);
    const int rc = pe_decode_jpeg(d.data(), (long long)d.size(), &w, &h, ref.data(), (long long)ref.size());
    if (pe_jpeg_read_coefs(d.data(), (long long)d.size(), buf.data(), n - 1) != -1) { printf("short cap accepted\n"); return 1; }
    const long long m = pe_jpeg_read_coefs(d.data(), (long long)d.size(), buf.data(), n);
    if ((rc == 0) != (m == n) || (rc != 0 && m != rc)) { printf("decode %d, coefs %lld (size %lld)\n", rc, m, n); return 1; }
    if (rc != 0) { rejected++; return 0; }
    if (pe_jpeg_coefs_to_bgr(buf.data(), got.data(), (long long)got.size()) != 0 || memcmp(ref.data(), got.data(), ref.size())) {
        printf("reconstruction differs from pe_decode_jpeg (%dx%d)\n", w, h);
        return 1;
    }
    ok++;
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    const int iters = atoi(argv[1]);
    uint64_t s = 123456789;
    auto rnd = [&]() { s = s * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(s >> 33); };
    long ok = 0, rejected = 0;
    int bad = 0;
    for (int a = 2; a < argc; a++) {
        const std::vector<uint8_t> base = slurp(argv[a]);
        if (base.size() < 16) return 2;
        for (size_t cut = 0; cut < base.size(); cut += 1 + base.size() / 64) bad += check(std::vector<uint8_t>(base.begin(), base.begin() + cut), ok, rejected);
        for (int it = 0; it < iters; it++) {
            std::vector<uint8_t> d = base;
            const int nm = 1 + rnd() % 6;
            for (int k = 0; k < nm; k++) {
                const int kind = rnd() % 4;
                if (kind == 0) d[rnd() % d.size()] = (uint8_t)rnd();
                else if (kind == 1) d[rnd() % d.size()] ^= (uint8_t)(1u << (rnd() % 8));
                else if (kind == 2 && d.size() > 16) d.resize(8 + rnd() % (d.size() - 8));
                else { const size_t p = rnd() % d.size(); d[p] = 0xFF; if (p + 1 < d.size()) d[p + 1] = (uint8_t)(0xC0 + rnd() % 0x20); }
            }
            bad += check(d, ok, rejected);
        }
        std::vector<uint8_t> junk(base.size());   // random bytes behind a JPEG signature
        for (auto& b : junk) b = (uint8_t)rnd();
        junk[0] = 0xFF; junk[1] = 0xD8;
        bad += check(junk, ok, rejected);
    }
    printf("accepted %ld rejected %ld mismatches %d\n", ok, rejected, bad);
    return bad ? 1 : 0;
}
