// Drives the group-FFT workers of integration/napi/snarkb200_napi.cc (groupFft, groupApplyKey) through the in-process N-API
// stand-in (tests/host/napi_stub/napi.h), linked against the real libsnarkb200.so.  Without a GPU the two exports must exist
// and createContext must report "no CUDA device"; with a GPU a 2^6-point G1 ifft and a batchApplyKey run through the
// addon's AsyncWorkers and are checked against the library called directly.
#include <cstdio>
#include "../../integration/napi/snarkb200_napi.cc"

static Napi::Value num(double v) { return Napi::Number::New(Napi::Env(), v); }
static Napi::Value bytes(const std::vector<uint8_t>& b) { return Napi::Uint8Array::New(Napi::Env(), b.data(), b.size()); }

int main() {
    Napi::Object ex = napi_stub_init();
    for (const char* n : {"groupFft", "groupApplyKey"})
        if (ex.Get(n).d->kind != Napi::Data::Function) { printf("export %s missing\n", n); return 1; }
    Napi::Value ctx = ex.Get("createContext").As<Napi::Function>().Call({num(0), num(0)});
    if (ctx.d->kind != Napi::Data::External) {
        if (Napi::Error::pending() != "snarkb200: no CUDA device") { printf("unexpected createContext failure: %s\n", Napi::Error::pending().c_str()); return 1; }
        printf("GROUP FFT SHIM CHECK PASSED (no CUDA device: createContext reported it; groupFft and groupApplyKey exported)\n");
        return 0;
    }
    sb_ctx* c = ctx.As<Napi::External<sb_ctx>>().Data();
    std::vector<uint8_t> pts(64 * 64), want(64 * 96), want2(64 * 64), one(32), inc(32, 0);
    if (sb_gen_points(c, SB_G1, 3, 64, pts.data()) || sb_fr_root(c, 0, one.data()) < 0 || sb_fr_root(c, 6, inc.data()) < 0) { printf("setup failed\n"); return 1; }
    if (sb_group_fft(c, SB_G1, pts.data(), 0, 64, 1, 1, want.data())) { printf("direct sb_group_fft failed\n"); return 1; }
    Napi::Value p = ex.Get("groupFft").As<Napi::Function>().Call({ctx, num(1), bytes(pts), num(0), num(1), num(1), num(32)});
    auto got = p.d->props.find("value");
    if (got == p.d->props.end() || got->second->bytes != want) { printf("groupFft through the addon differs\n"); return 1; }
    if (sb_group_batch_apply_key(c, SB_G1, pts.data(), 0, 64, one.data(), inc.data(), 0, want2.data())) { printf("direct apply key failed\n"); return 1; }
    p = ex.Get("groupApplyKey").As<Napi::Function>().Call({ctx, num(1), bytes(pts), bytes(one), bytes(inc), num(0), num(0), num(32)});
    got = p.d->props.find("value");
    if (got == p.d->props.end() || got->second->bytes != want2) { printf("groupApplyKey through the addon differs\n"); return 1; }
    p = ex.Get("groupFft").As<Napi::Function>().Call({ctx, num(1), bytes(std::vector<uint8_t>(3 * 64)), num(0), num(0), num(0), num(32)});
    if (p.d->props.find("error") == p.d->props.end()) { printf("a 3-point group fft was not rejected\n"); return 1; }
    printf("GROUP FFT SHIM CHECK PASSED (GPU: groupFft, groupApplyKey and the error path through the addon)\n");
    return 0;
}
