// The test double of stub_engine.cpp plus the calibration calls of include/poseengine.h (pe_calibrate_begin / _end,
// pe_calibration_get / _set), for tests/test_calibration_cli.py.  One translation unit: the calls below use the stub's engine
// handle, log and error helpers.  TEST INFRASTRUCTURE: nothing here is shipped.
//   STUB_CALIB_CHANGED  "3,1,0": what the k-th pe_calibrate_end of the process reports (0 past the list)
// pe_calibration_get returns a fixed table of six layers; pe_calibration_set refuses text that is not a table.
#include "stub_engine.cpp"

extern "C" {
int pe_calibrate_begin(pe_engine* e) {
    Exclusive x(e);
    logf("calibrate_begin engine=%d", e->id);
    return PE_OK;
}
int pe_calibrate_end(pe_engine* e, int* changed) {
    Exclusive x(e);
    static std::atomic<int> calls{0};
    const int k = calls++;
    int v = 0;
    std::string list = getenv("STUB_CALIB_CHANGED") ? getenv("STUB_CALIB_CHANGED") : "";
    for (int i = 0; i <= k && !list.empty(); i++) {
        const size_t comma = list.find(',');
        v = i == k ? atoi(list.substr(0, comma).c_str()) : 0;
        list = comma == std::string::npos ? "" : list.substr(comma + 1);
    }
    *changed = v;
    logf("calibrate_end engine=%d changed=%d", e->id, v);
    return PE_OK;
}
int pe_calibration_get(const pe_engine* e, char* buf, int cap) {
    char text[256];
    snprintf(text, sizeof text, "pe_calibration 1\nprecision %d\nweights 0123456789abcdef\nlayer conv0 s8 -3\nlayer conv1 s8 2\nlayer conv2 s8 1\n"
             "layer conv3 s8 0\nlayer conv4 s8 -1\nlayer conv5 s8 4\n", e->cfg.precision);
    const int n = (int)strlen(text);
    if (buf && n < cap) memcpy(buf, text, n + 1);
    logf("calibration_get engine=%d", e->id);
    return n;
}
int pe_calibration_set(pe_engine* e, const char* text) {
    Exclusive x(e);
    if (strncmp(text, "pe_calibration ", 15) != 0) return fail(e, PE_ERR_INVALID, "stub: calibration table line 1: not a calibration table");
    const std::string first(text, strcspn(text, "\n"));
    logf("calibration_set engine=%d bytes=%d first=%s", e->id, (int)strlen(text), first.c_str());
    return PE_OK;
}
}
