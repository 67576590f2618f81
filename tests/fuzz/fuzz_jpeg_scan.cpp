// Mutation fuzzer for scan images (pe_jpeg_read_scan) and the host run of the GPU entropy decoder (pe_jpeg_scan_to_coefs_host).
// Built with -fsanitize=address,undefined by tests/test_jpeg_scan.py; any finding aborts.  On every mutated stream it checks that
// the scan stage returns pe_jpeg_read_coefs's code (or -3 for a stream that needs the host entropy stage), and that the coefficient
// image decoded from an accepted scan image equals pe_jpeg_read_coefs's at several subsequence lengths, with the data error flagged
// exactly where pe_jpeg_read_coefs rejects the file.
// usage: fuzz_jpeg_scan <iterations> <file.jpg>...
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
static int check(const std::vector<uint8_t>& d, long& decoded, long& flagged, long& rejected) {
    const long long size = (long long)d.size();
    const long long nc = pe_jpeg_read_coefs(d.data(), size, nullptr, 0);
    if (nc > 64000000) { rejected++; return 0; }
    std::vector<uint8_t> ref(nc > 0 ? (size_t)nc : 0);
    const long long rc = nc > 0 ? pe_jpeg_read_coefs(d.data(), size, ref.data(), nc) : nc;
    const long long ns = pe_jpeg_read_scan(d.data(), size, nullptr, 0);
    if (ns == -3) { rejected++; return 0; }
    if (ns < 0) {
        if (ns != rc) { printf("scan %lld, coefs %lld\n", ns, rc); return 1; }
        rejected++;
        return 0;
    }
    if (rc != nc && rc != -1) { printf("scan accepted, coefs %lld\n", rc); return 1; }
    std::vector<uint8_t> scan((size_t)ns);   // exact sizes: ASAN sees any access past them
    if (pe_jpeg_read_scan(d.data(), size, scan.data(), ns - 1) != -1) { printf("short cap accepted\n"); return 1; }
    if (pe_jpeg_read_scan(d.data(), size, scan.data(), ns) != ns) { printf("second read differs\n"); return 1; }
    long long total = 0;
    memcpy(&total, scan.data() + 24, 8);   // pe_jpeg_coef_header.total_bytes
    if (total <= 0 || total > 64000000 || (nc > 0 && total != nc)) { printf("coefficient size %lld vs %lld\n", total, nc); return 1; }
    std::vector<uint8_t> got((size_t)total);
    const int subseq[3] = {32, 1000, 1 << 30};
    for (int S : subseq) {
        const long long r = pe_jpeg_scan_to_coefs_host(scan.data(), got.data(), total, S);
        if (rc == nc ? (r != nc || memcmp(got.data(), ref.data(), (size_t)nc)) : r != -4) {
            printf("subsequences of %d bits: host run %lld, coefs %lld\n", S, r, rc);
            return 1;
        }
    }
    if (rc == nc) decoded++; else flagged++;
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 3) return 2;
    const int iters = atoi(argv[1]);
    uint64_t s = 987654321;
    auto rnd = [&]() { s = s * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(s >> 33); };
    long decoded = 0, flagged = 0, rejected = 0;
    int bad = 0;
    for (int a = 2; a < argc; a++) {
        const std::vector<uint8_t> base = slurp(argv[a]);
        if (base.size() < 16) return 2;
        for (size_t cut = 0; cut < base.size(); cut += 1 + base.size() / 64)
            bad += check(std::vector<uint8_t>(base.begin(), base.begin() + cut), decoded, flagged, rejected);
        for (int it = 0; it < iters; it++) {
            std::vector<uint8_t> d = base;
            const int nm = 1 + rnd() % 6;
            for (int k = 0; k < nm; k++) {
                const int kind = rnd() % 5;
                if (kind == 0) d[rnd() % d.size()] = (uint8_t)rnd();
                else if (kind == 1) d[rnd() % d.size()] ^= (uint8_t)(1u << (rnd() % 8));
                else if (kind == 2 && d.size() > 16) d.resize(8 + rnd() % (d.size() - 8));
                else if (kind == 3) { const size_t p = rnd() % d.size(); d[p] = 0xFF; if (p + 1 < d.size()) d[p + 1] = (uint8_t)(0xC0 + rnd() % 0x20); }
                else { const size_t p = rnd() % d.size(); d[p] = 0xFF; if (p + 1 < d.size()) d[p + 1] = (uint8_t)(0xD0 + rnd() % 8); }   // RST
            }
            bad += check(d, decoded, flagged, rejected);
        }
    }
    printf("decoded %ld flagged %ld rejected %ld mismatches %d\n", decoded, flagged, rejected, bad);
    return bad ? 1 : 0;
}
