"""The engine's owning buffers (csrc/buffers.h) without a GPU: a driver under ASAN + UBSan links its own cudaMalloc / cudaFree /
cudaMallocHost / cudaFreeHost, which fail on demand and count the live blocks, and checks what each call leaves behind."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "caffe_rtpose_b200", "csrc")

DRIVER = r"""
#include "buffers.h"
#include <stdio.h>
#include <stdlib.h>
#include <set>
#include <utility>
#include <vector>

// cudart stand-ins: every block is recorded, so a double or unknown free and a leak are seen
static std::set<void*> live;
static int fail_next = 0;
static long allocs = 0;
static cudaError_t fake_alloc(void** p, size_t n) {
    if (fail_next) { fail_next = 0; *p = (void*)0x40; return cudaErrorMemoryAllocation; }   // a failed call may leave *p set
    if (posix_memalign(p, 256, n ? n : 1)) return cudaErrorMemoryAllocation;
    live.insert(*p);
    allocs++;
    return cudaSuccess;
}
static cudaError_t fake_free(void* p) {
    if (!p) return cudaSuccess;
    if (!live.erase(p)) { printf("FAIL free of a pointer that is not live\n"); exit(1); }
    free(p);
    return cudaSuccess;
}
extern "C" cudaError_t cudaMalloc(void** p, size_t n) { return fake_alloc(p, n); }
extern "C" cudaError_t cudaMallocHost(void** p, size_t n) { return fake_alloc(p, n); }
extern "C" cudaError_t cudaFree(void* p) { return fake_free(p); }
extern "C" cudaError_t cudaFreeHost(void* p) { return fake_free(p); }

static bool report(const char* name, bool ok) { printf("%s %s\n", ok ? "PASS" : "FAIL", name); return ok; }

template <class B> static void check(const char* kind) {
    char name[128];
    {
        B b;
        bool ok = b.reserve(1000) == cudaSuccess && b.get() && b.size() == 1000;
        fail_next = 1;
        ok = ok && b.reserve(2000) == cudaErrorMemoryAllocation && b.get() == nullptr && b.size() == 0;
        snprintf(name, sizeof name, "%s_failed_reserve_leaves_empty", kind);
        report(name, ok && live.empty());
        const long before = allocs;   // a smaller request than the lost buffer's must allocate again, not return null
        ok = b.reserve(500) == cudaSuccess && b.get() && b.size() == 500 && allocs == before + 1;
        snprintf(name, sizeof name, "%s_smaller_reserve_after_failure_allocates", kind);
        report(name, ok);
    }
    {
        B b;
        b.reserve(4096);
        void* p = b.get();
        const long before = allocs;
        const bool ok = b.reserve(4096) == cudaSuccess && b.reserve(1) == cudaSuccess && b.reserve(0) == cudaSuccess && b.get() == p &&
                        b.size() == 4096 && allocs == before;
        snprintf(name, sizeof name, "%s_fitting_reserve_keeps_buffer", kind);
        report(name, ok);
        const bool grown = b.reserve(8192) == cudaSuccess && b.size() == 8192 && live.size() == 1;
        snprintf(name, sizeof name, "%s_growing_reserve_frees_old", kind);
        report(name, grown);
    }
    {
        B a;
        a.reserve(64);
        void* p = a.get();
        B b(std::move(a));
        bool ok = a.get() == nullptr && a.size() == 0 && b.get() == p && b.size() == 64;
        std::vector<B> v(1);   // relocation on growth moves every element
        v[0].reserve(32);
        void* q = v[0].get();
        for (int i = 0; i < 40; i++) v.emplace_back().reserve(8);
        ok = ok && v[0].get() == q && live.size() == 42;
        snprintf(name, sizeof name, "%s_move_leaves_source_empty", kind);
        report(name, ok);
    }
    {
        B b;
        const size_t counts[] = {1, 0, 300, 257, 4096, 3};
        std::vector<std::pair<char*, size_t>> r;
        auto layout = [&](pe::Carver& k) {
            r.clear();
            r.push_back({k.take<char>(counts[0]), counts[0]});
            r.push_back({(char*)k.take<double>(counts[1]), counts[1] * 8});
            r.push_back({(char*)k.take<int>(counts[2]), counts[2] * 4});
            r.push_back({(char*)k.take<short>(counts[3]), counts[3] * 2});
            r.push_back({k.take<char>(counts[4]), counts[4]});
            r.push_back({(char*)k.take<float>(counts[5]), counts[5] * 4});
        };
        bool ok = pe::reserve_carved(b, layout) == cudaSuccess && b.get();
        char* base = (char*)b.get();
        for (size_t i = 0; ok && i < r.size(); i++) {
            ok = ((size_t)r[i].first % 256) == 0 && r[i].first >= base && r[i].first + r[i].second <= base + b.size();
            if (i) ok = ok && r[i].first >= r[i - 1].first + r[i - 1].second;   // in order, so no two ranges overlap
        }
        snprintf(name, sizeof name, "%s_carved_ranges_aligned_and_disjoint", kind);
        report(name, ok);
        const long before = allocs;   // a second layout over a buffer that fits reuses it
        ok = pe::reserve_carved(b, layout) == cudaSuccess && r[0].first == base && allocs == before;
        B c;
        fail_next = 1;
        ok = ok && pe::reserve_carved(c, layout) == cudaErrorMemoryAllocation && c.get() == nullptr && c.size() == 0;
        for (auto& x : r) ok = ok && x.first == nullptr;
        snprintf(name, sizeof name, "%s_failed_carve_hands_out_null", kind);
        report(name, ok);
    }
}

int main() {
    check<pe::DeviceBuffer>("device");
    check<pe::PinnedBuffer>("pinned");
    report("no_block_live_at_exit", live.empty());
    return 0;
}
"""

CHECKS = ["failed_reserve_leaves_empty", "smaller_reserve_after_failure_allocates", "fitting_reserve_keeps_buffer",
          "growing_reserve_frees_old", "move_leaves_source_empty", "carved_ranges_aligned_and_disjoint", "failed_carve_hands_out_null"]


@pytest.fixture(scope="module")
def results(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ not found")
    d = tmp_path_factory.mktemp("buffers")
    src, exe = d / "buffers_driver.cpp", d / "buffers_driver"
    src.write_text(DRIVER)
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Werror", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                        "-I", CSRC, "-I", "/usr/local/cuda/include", str(src), "-o", str(exe)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.stdout[-2000:], r.stderr[-3000:])
    return dict(reversed(line.split(" ", 1)) for line in r.stdout.splitlines())


@pytest.mark.parametrize("kind", ["device", "pinned"])
@pytest.mark.parametrize("check", CHECKS)
def test_buffer(results, kind, check):
    assert results.get(kind + "_" + check) == "PASS", results


def test_no_block_live_at_exit(results):
    assert results.get("no_block_live_at_exit") == "PASS", results
