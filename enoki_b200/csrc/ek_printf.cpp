/*
 * ek_printf.cpp -- the format rules of cuda_printf (ek_trace_printf): the parser that checks a format against the
 * types of its arguments when the print is recorded, and the host formatter that writes one line per element after
 * the evaluation that computed the arguments.  No other module parses formats.
 *
 * The reference hands its format to the device's vprintf unchecked (jit.cu:863-916); here a format is accepted only
 * when every conversion has a C meaning for the argument it consumes, so that the host can format it with snprintf:
 *   %%, flags "-+ #0", a width and a ".precision" given as digits, the length modifiers hh / h / l / ll,
 *   the integer conversions d i u o x X c (integer, Bool and pointer arguments; %c takes no length modifier) and
 *   the float conversions f F e E g G a A (Float32 / Float64 arguments; length modifier l or none).
 */
#include "ek_internal.h"
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace {

const uint32_t EK_PRINTF_MAX_FIELD = 4096;     /* largest width / precision accepted */

bool is_int_conv(char c) { return c && strchr("diuoxXc", c) != nullptr; }
bool is_float_conv(char c) { return c && strchr("fFeEgGaA", c) != nullptr; }
bool is_signed_conv(char c) { return c == 'd' || c == 'i' || c == 'c'; }

const char *len_name(uint8_t len) {
    static const char *names[] = { "", "hh", "h", "l", "ll" };
    return names[len];
}

std::string arg_desc(uint32_t k, const ek_type *types, uint32_t narg) {
    if (k >= narg) return "no argument (" + std::to_string(narg) + " given)";
    return "argument " + std::to_string(k + 1) + " of type " + ek_type_name(types[k]);
}

} // namespace

bool ek_printf_parse(const char *fmt, uint32_t narg, const ek_type *types, std::vector<EkPrintSeg> &segs,
                     std::string &err) {
    segs.clear();
    if (!fmt) { err = "ek_trace_printf(): the format is NULL"; return false; }
    for (uint32_t k = 0; k < narg; ++k) {
        if (types[k] == EK_FLOAT16) { err = "ek_trace_printf(): argument " + std::to_string(k + 1) + " has type f16, which cannot be printed"; return false; }
        if (ek_type_size(types[k]) == 0) { err = "ek_trace_printf(): argument " + std::to_string(k + 1) + " has an invalid type"; return false; }
    }
    std::string text;
    uint32_t nconv = 0;
    const char *p = fmt;
    while (*p) {
        if (*p != '%') { text += *p++; continue; }
        const char *start = p++;
        if (*p == '%') { text += '%'; ++p; continue; }
        if (!*p) { err = "ek_trace_printf(): the format ends with a lone '%'"; return false; }
        while (*p && strchr("-+ #0", *p)) ++p;
        auto digits = [&](const char *what) -> bool {
            uint32_t v = 0;
            while (*p >= '0' && *p <= '9') {
                v = v * 10 + (uint32_t) (*p++ - '0');
                if (v > EK_PRINTF_MAX_FIELD) {
                    err = std::string("ek_trace_printf(): ") + what + " in conversion '" + std::string(start, p) +
                          "...' exceeds " + std::to_string(EK_PRINTF_MAX_FIELD);
                    return false;
                }
            }
            if (*p == '*') {
                err = std::string("ek_trace_printf(): a '*' ") + what + " in conversion '" + std::string(start, p + 1) +
                      "' is not supported (" + arg_desc(nconv, types, narg) + ")";
                return false;
            }
            return true;
        };
        if (!digits("width")) return false;
        if (*p == '.') { ++p; if (!digits("precision")) return false; }
        uint8_t len = 0;
        if (p[0] == 'h' && p[1] == 'h') { len = 1; p += 2; }
        else if (p[0] == 'h') { len = 2; p += 1; }
        else if (p[0] == 'l' && p[1] == 'l') { len = 4; p += 2; }
        else if (p[0] == 'l') { len = 3; p += 1; }
        const char conv = *p;
        const std::string spec(start, conv ? p + 1 : p);
        if (!conv) { err = "ek_trace_printf(): the format ends inside conversion '" + spec + "'"; return false; }
        ++p;
        const uint32_t k = nconv++;
        const std::string what = "ek_trace_printf(): conversion '" + spec + "' ";
        if (!is_int_conv(conv) && !is_float_conv(conv)) { err = what + "is not supported (" + arg_desc(k, types, narg) + ")"; return false; }
        if (k >= narg) { err = what + "has " + arg_desc(k, types, narg); return false; }
        const ek_type t = types[k];
        if (is_float_conv(conv)) {
            if (t != EK_FLOAT32 && t != EK_FLOAT64) { err = what + "takes a Float32 / Float64 value, not " + arg_desc(k, types, narg); return false; }
            if (len != 0 && len != 3) { err = what + "does not accept the length modifier '" + len_name(len) + "' (" + arg_desc(k, types, narg) + ")"; return false; }
        } else {
            if (ek_is_float(t)) { err = what + "takes an integer, Bool or pointer value, not " + arg_desc(k, types, narg); return false; }
            if (conv == 'c' && len != 0) { err = what + "does not accept the length modifier '" + len_name(len) + "' (" + arg_desc(k, types, narg) + ")"; return false; }
        }
        if (!text.empty()) { segs.push_back({ text, 0, 0, 0 }); text.clear(); }
        segs.push_back({ spec, conv, len, (uint8_t) k });
    }
    if (nconv != narg) {
        err = "ek_trace_printf(): the format has " + std::to_string(nconv) + " conversion(s) for " + std::to_string(narg) + " argument(s)";
        return false;
    }
    if (!text.empty()) segs.push_back({ text, 0, 0, 0 });
    return true;
}

/* Float32 is widened to double exactly (the reference's cvt.f64.f32); integers are converted to the C type that the
   conversion and its length modifier name, as C converts a value of the argument's type to it. */
void ek_printf_append(std::string &out, const std::vector<EkPrintSeg> &segs, const ek_type *types, const uint64_t *bits) {
    char buf[256];
    for (const EkPrintSeg &s : segs) {
        if (!s.conv) { out += s.text; continue; }
        const ek_type t = types[s.arg];
        const uint64_t b = bits[s.arg];
        const char *f = s.text.c_str();
        auto put = [&](auto value) {
            int n = snprintf(buf, sizeof(buf), f, value);
            if (n < 0) return;
            if ((size_t) n < sizeof(buf)) { out.append(buf, (size_t) n); return; }
            size_t at = out.size();
            out.resize(at + (size_t) n + 1);
            snprintf(&out[at], (size_t) n + 1, f, value);
            out.resize(at + (size_t) n);
        };
        if (is_float_conv(s.conv)) {
            double d;
            if (t == EK_FLOAT32) { float x; uint32_t w = (uint32_t) b; memcpy(&x, &w, 4); d = (double) x; }
            else memcpy(&d, &b, 8);
            put(d);
            continue;
        }
        /* the argument's value, sign- or zero-extended to 64 bits */
        uint64_t ext;
        switch (t) {
            case EK_INT8:  ext = (uint64_t) (int64_t) (int8_t) b; break;
            case EK_INT16: ext = (uint64_t) (int64_t) (int16_t) b; break;
            case EK_INT32: ext = (uint64_t) (int64_t) (int32_t) b; break;
            case EK_UINT8: ext = (uint8_t) b; break;
            case EK_UINT16: ext = (uint16_t) b; break;
            case EK_UINT32: ext = (uint32_t) b; break;
            case EK_BOOL: ext = (b & 0xffu) != 0; break;
            default: ext = b; break;                      /* Int64, UInt64, Pointer */
        }
        if (is_signed_conv(s.conv)) {
            if (s.len == 3) put((long) (int64_t) ext);
            else if (s.len == 4) put((long long) (int64_t) ext);
            else put((int) (int64_t) ext);
        } else {
            if (s.len == 3) put((unsigned long) ext);
            else if (s.len == 4) put((unsigned long long) ext);
            else put((unsigned) ext);
        }
    }
}
