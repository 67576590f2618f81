// Calibration table text (calib_table.h): writer and checking reader.  No CUDA: tests/fuzz/fuzz_calibration_table.cpp builds it alone.
#include "calib_table.h"

#include <ctype.h>
#include <errno.h>
#include <stdio.h>
#include <stdlib.h>

#include <map>
#include <sstream>

namespace pe {

std::string write_calibration_table(const CalibTable& t) {
    std::string s;
    char buf[320];
    snprintf(buf, sizeof buf, "pe_calibration %d\nprecision %d\nweights %016llx\n", CALIB_TABLE_VERSION, t.precision, (unsigned long long)t.weights);
    s += buf;
    for (const CalibLayer& l : t.layers) s += "layer " + l.name + " " + l.kind + " " + std::to_string(l.log2_scale) + "\n";
    return s;
}

// a decimal integer that is the whole token and fits an int
static bool parse_int(const std::string& tok, int& v) {
    if (tok.empty() || tok.size() > 12) return false;
    for (size_t i = 0; i < tok.size(); i++)
        if (!(isdigit((unsigned char)tok[i]) || (i == 0 && (tok[i] == '-' || tok[i] == '+') && tok.size() > 1))) return false;
    errno = 0;
    const long long x = strtoll(tok.c_str(), nullptr, 10);
    if (errno || x < -2147483647LL || x > 2147483647LL) return false;
    v = (int)x;
    return true;
}

static bool parse_hex64(const std::string& tok, uint64_t& v) {
    if (tok.size() != 16) return false;
    v = 0;
    for (char c : tok) {
        const int d = c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1;
        if (d < 0) return false;
        v = v << 4 | (uint64_t)d;
    }
    return true;
}

int read_calibration_table(const char* text, const CalibTable& expect, std::vector<int>& log2_out, std::string& err) {
    if (!text) { err = "null calibration table"; return -1; }
    auto bad = [&](int line, const std::string& what) { err = "calibration table line " + std::to_string(line) + ": " + what; return -1; };
    // the lines that carry a fact: tokens without the comment
    struct Line { int no; std::vector<std::string> tok; };
    std::vector<Line> lines;
    {
        int no = 0;
        for (const char* p = text; *p;) {
            const char* e = p;
            while (*e && *e != '\n') e++;
            no++;
            std::string s(p, e - p);
            const size_t hash = s.find('#');
            if (hash != std::string::npos) s.resize(hash);
            Line l{no, {}};
            std::istringstream in(s);
            for (std::string t; in >> t;) l.tok.push_back(t);
            if (!l.tok.empty()) lines.push_back(std::move(l));
            p = *e ? e + 1 : e;
        }
    }
    if (lines.empty()) { err = "empty calibration table"; return -1; }
    size_t k = 0;
    auto header = [&](const char* key, std::string& val) -> int {
        if (k >= lines.size()) { err = std::string("calibration table ends before its '") + key + "' line"; return -1; }
        const Line& l = lines[k++];
        if (l.tok[0] != key) return bad(l.no, "expected '" + std::string(key) + " ...', found '" + l.tok[0] + "'");
        if (l.tok.size() != 2) return bad(l.no, l.tok.size() < 2 ? "'" + std::string(key) + "' without a value" : "trailing text '" + l.tok[2] + "'");
        val = l.tok[1];
        return 0;
    };
    std::string v;
    int iv = 0;
    if (header("pe_calibration", v)) return -1;
    if (!parse_int(v, iv)) return bad(lines[k - 1].no, "version '" + v + "' is not an integer");
    if (iv != CALIB_TABLE_VERSION) return bad(lines[k - 1].no, "calibration table version " + v + ": this library reads version " + std::to_string(CALIB_TABLE_VERSION));
    if (header("precision", v)) return -1;
    if (!parse_int(v, iv)) return bad(lines[k - 1].no, "precision '" + v + "' is not an integer");
    if (iv != expect.precision)
        return bad(lines[k - 1].no, "the table is for precision " + v + ", the engine runs precision " + std::to_string(expect.precision));
    if (header("weights", v)) return -1;
    uint64_t wh = 0;
    if (!parse_hex64(v, wh)) return bad(lines[k - 1].no, "weights hash '" + v + "' is not 16 hex digits");
    if (wh != expect.weights) {
        char b[160];
        snprintf(b, sizeof b, "the table was calibrated with other weights (hash %016llx, the engine's %016llx)", (unsigned long long)wh,
                 (unsigned long long)expect.weights);
        return bad(lines[k - 1].no, b);
    }
    std::map<std::string, size_t> index;   // engine layer -> position
    for (size_t j = 0; j < expect.layers.size(); j++) index[expect.layers[j].name] = j;
    std::map<std::string, int> seen;       // table layer -> its line
    std::vector<int> out(expect.layers.size(), 0);
    size_t j = 0;
    for (; k < lines.size(); k++, j++) {
        const Line& l = lines[k];
        if (l.tok[0] != "layer") return bad(l.no, "expected 'layer <name> <kind> <log2 scale>', found '" + l.tok[0] + "'");
        if (l.tok.size() < 4) return bad(l.no, "'layer' needs a name, a stored kind and a log2 scale");
        if (l.tok.size() > 4) return bad(l.no, "trailing text '" + l.tok[4] + "'");
        const std::string& name = l.tok[1];
        const auto it = index.find(name);
        if (it == index.end()) return bad(l.no, "unknown layer " + name + ": the engine has no conv layer of that name that stores an activation");
        if (seen.count(name)) return bad(l.no, "layer " + name + " appears twice (first on line " + std::to_string(seen[name]) + ")");
        seen[name] = l.no;
        if (it->second != j) {
            if (it->second > j) {   // a layer the engine runs before this one is not here (yet)
                const std::string& want = expect.layers[j].name;
                bool later = false;
                for (size_t q = k + 1; q < lines.size() && !later; q++) later = lines[q].tok.size() > 1 && lines[q].tok[0] == "layer" && lines[q].tok[1] == want;
                if (!later) { err = "calibration table: layer " + want + " is missing (expected before line " + std::to_string(l.no) + ")"; return -1; }
            }
            return bad(l.no, "layer " + name + " is out of order: the engine runs " + expect.layers[j].name + " here");
        }
        if (l.tok[2] != expect.layers[j].kind)
            return bad(l.no, "layer " + name + " stores " + l.tok[2] + " in the table, " + expect.layers[j].kind +
                                 " in the engine (another f16_layers list or precision)");
        int e2 = 0;
        if (!parse_int(l.tok[3], e2)) return bad(l.no, "layer " + name + ": log2 scale '" + l.tok[3] + "' is not an integer");
        if (e2 < -CALIB_MAX_LOG2 || e2 > CALIB_MAX_LOG2)
            return bad(l.no, "layer " + name + ": log2 scale " + l.tok[3] + " is outside [-100, 100]");
        out[j] = e2;
    }
    if (j < expect.layers.size()) { err = "calibration table: layer " + expect.layers[j].name + " is missing (the table ends before it)"; return -1; }
    log2_out.swap(out);
    return 0;
}

}  // namespace pe
