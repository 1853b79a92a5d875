// snarkb200_napi.cc — N-API addon binding libsnarkb200.so's C ABI (include/snarkb200.h) for Node.js.
// Not built for Node by this repository's build or tests (they need no node / node-addon-api headers); it is the binding a
// snarkjs maintainer adds, see INTEGRATION.md.  Build with node-gyp (binding.gyp next to this file).  What IS checked here:
// tests/test_abi.py compiles this file against an in-process stand-in for the N-API classes it uses
// (tests/host/napi_stub/napi.h), links it against the real libsnarkb200.so and drives it (tests/host/napi_shim_check.cpp).
//
// Concurrency: overlapping calls on one context are safe — libsnarkb200 locks the context for the duration of every entry
// (snarkb200.h "threading"), so AsyncWorkers that land on different libuv threads (joinABC queues one task per 2^22
// elements before awaiting them, src/groth16_prove.js:328-360) run one after the other instead of racing.
//
// Every bulk call runs in a Napi::AsyncWorker so the event loop is never blocked — the reference's methods are async
// (build/snarkjs.js:14196-14232) — and resolves/rejects a Promise; errors carry sb_last_error() so that messages match
// the reference's `throw new Error(...)`.
#include <napi.h>
#include <vector>
#include "snarkb200.h"

namespace {

sb_ctx* ctx_of(const Napi::Value& v) { return v.As<Napi::External<sb_ctx>>().Data(); }

Napi::Value Create(const Napi::CallbackInfo& info) {
  sb_ctx* c = nullptr;
  int rc = sb_create(info[0].As<Napi::Number>().Int32Value(), info[1].As<Napi::Number>().Int32Value(), &c);
  if (rc) {
    Napi::Error::New(info.Env(), rc == SB_ERR_NODEVICE ? "snarkb200: no CUDA device" : "snarkb200: sb_create failed").ThrowAsJavaScriptException();
    return info.Env().Undefined();
  }
  return Napi::External<sb_ctx>::New(info.Env(), c, [](Napi::Env, sb_ctx* p) { sb_destroy(p); });
}

// Generic worker: `fn` runs off the event loop and fills `out`; inputs are kept alive by references.
class Worker : public Napi::AsyncWorker {
 public:
  using Fn = std::function<int(std::vector<uint8_t>&)>;
  Worker(Napi::Env env, sb_ctx* c, size_t out_len, Fn fn, std::vector<Napi::Reference<Napi::Uint8Array>> keep)
      : Napi::AsyncWorker(env), deferred(Napi::Promise::Deferred::New(env)), c_(c), out_(out_len), fn_(std::move(fn)), keep_(std::move(keep)) {}
  void Execute() override { if (fn_(out_) != 0) SetError(sb_last_error(c_)); }
  void OnOK() override { deferred.Resolve(Napi::Buffer<uint8_t>::Copy(Env(), out_.data(), out_.size())); }
  void OnError(const Napi::Error& e) override { deferred.Reject(e.Value()); }
  Napi::Promise::Deferred deferred;
 private:
  sb_ctx* c_; std::vector<uint8_t> out_; Fn fn_; std::vector<Napi::Reference<Napi::Uint8Array>> keep_;
};

Napi::Value Queue(Napi::Env env, sb_ctx* c, size_t out_len, Worker::Fn fn, std::initializer_list<Napi::Uint8Array> inputs) {
  std::vector<Napi::Reference<Napi::Uint8Array>> keep;
  for (auto& a : inputs) keep.push_back(Napi::Persistent(a));
  auto* w = new Worker(env, c, out_len, std::move(fn), std::move(keep));
  w->Queue();
  return w->deferred.Promise();
}

// multiExpAffine(ctx, group, bases, scalars, n8q) -> Promise<Buffer(3*n8q*group)>     (build/snarkjs.js:14666-14668)
Napi::Value MultiExpAffine(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]);
  int group = info[1].As<Napi::Number>().Int32Value();
  auto bases = info[2].As<Napi::Uint8Array>(); auto scalars = info[3].As<Napi::Uint8Array>();
  size_t n8q = info[4].As<Napi::Number>().Uint32Value();
  size_t n = bases.ByteLength() / (2 * n8q * group);
  uint32_t ss = n ? (uint32_t)(scalars.ByteLength() / n) : 0;    // divisibility is checked by the JS wrapper
  const uint8_t* pb = bases.Data(); const uint8_t* ps = scalars.Data();
  return Queue(info.Env(), c, 3 * n8q * group, [=](std::vector<uint8_t>& out) {
    return group == 1 ? sb_msm_g1_affine(c, pb, ps, ss, n, out.data()) : sb_msm_g2_affine(c, pb, ps, ss, n, out.data());
  }, {bases, scalars});
}

// nttFr(ctx, buff, inverse) -> Promise<Buffer>                                          (15101-15107)
Napi::Value NttFr(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); auto buff = info[1].As<Napi::Uint8Array>(); int inverse = info[2].As<Napi::Number>().Int32Value();
  size_t n = buff.ByteLength() / 32; const uint8_t* p = buff.Data();
  return Queue(info.Env(), c, buff.ByteLength(), [=](std::vector<uint8_t>& out) { return sb_ntt_fr(c, p, n, inverse, out.data()); }, {buff});
}

// frBatchApplyKey(ctx, buff, first, inc)                                                 (14273-14384)
Napi::Value FrBatchApplyKey(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); auto buff = info[1].As<Napi::Uint8Array>(); auto first = info[2].As<Napi::Uint8Array>(); auto inc = info[3].As<Napi::Uint8Array>();
  size_t n = buff.ByteLength() / 32; const uint8_t *p = buff.Data(), *pf = first.Data(), *pi = inc.Data();
  return Queue(info.Env(), c, buff.ByteLength(), [=](std::vector<uint8_t>& out) { return sb_fr_batch_apply_key(c, p, n, pf, pi, out.data()); }, {buff, first, inc});
}

// frConvert(ctx, buff, toMontgomery)                                                     (12895-12896)
Napi::Value FrConvert(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); auto buff = info[1].As<Napi::Uint8Array>(); int to = info[2].As<Napi::Number>().Int32Value();
  size_t n = buff.ByteLength() / 32; const uint8_t* p = buff.Data();
  return Queue(info.Env(), c, buff.ByteLength(), [=](std::vector<uint8_t>& out) {
    return to ? sb_fr_batch_to_montgomery(c, p, n, out.data()) : sb_fr_batch_from_montgomery(c, p, n, out.data());
  }, {buff});
}

// qapJoinAbc(ctx, a, b, c)                                                               (src/groth16_prove.js:320-374)
Napi::Value QapJoinAbc(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); auto a = info[1].As<Napi::Uint8Array>(); auto b = info[2].As<Napi::Uint8Array>(); auto cc = info[3].As<Napi::Uint8Array>();
  size_t n = a.ByteLength() / 32; const uint8_t *pa = a.Data(), *pb = b.Data(), *pc = cc.Data();
  return Queue(info.Env(), c, a.ByteLength(), [=](std::vector<uint8_t>& out) { return sb_qap_join_abc(c, pa, pb, pc, n, out.data()); }, {a, b, cc});
}

// groupFft(ctx, group, buff, inJacobian, inverse, outJacobian, n8q) -> Promise<Buffer>     (G.fft / G.ifft 15101-15107)
Napi::Value GroupFft(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); int group = info[1].As<Napi::Number>().Int32Value(); auto buff = info[2].As<Napi::Uint8Array>();
  int in_jac = info[3].As<Napi::Number>().Int32Value(), inverse = info[4].As<Napi::Number>().Int32Value(), out_jac = info[5].As<Napi::Number>().Int32Value();
  size_t n8 = info[6].As<Napi::Number>().Uint32Value() * group;
  size_t n = buff.ByteLength() / ((in_jac ? 3 : 2) * n8); const uint8_t* p = buff.Data();
  return Queue(info.Env(), c, n * (out_jac ? 3 : 2) * n8, [=](std::vector<uint8_t>& out) {
    return sb_group_fft(c, group, p, in_jac, n, inverse, out_jac, out.data());
  }, {buff});
}

// groupApplyKey(ctx, group, buff, first, inc, inJacobian, outJacobian, n8q) -> Promise<Buffer>   (G.batchApplyKey 14268-14385)
Napi::Value GroupApplyKey(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); int group = info[1].As<Napi::Number>().Int32Value(); auto buff = info[2].As<Napi::Uint8Array>();
  auto first = info[3].As<Napi::Uint8Array>(); auto inc = info[4].As<Napi::Uint8Array>();
  int in_jac = info[5].As<Napi::Number>().Int32Value(), out_jac = info[6].As<Napi::Number>().Int32Value();
  size_t n8 = info[7].As<Napi::Number>().Uint32Value() * group;
  size_t n = buff.ByteLength() / ((in_jac ? 3 : 2) * n8); const uint8_t *p = buff.Data(), *pf = first.Data(), *pi = inc.Data();
  return Queue(info.Env(), c, n * (out_jac ? 3 : 2) * n8, [=](std::vector<uint8_t>& out) {
    return sb_group_batch_apply_key(c, group, p, in_jac, n, pf, pi, out_jac, out.data());
  }, {buff, first, inc});
}

// groth16Load(ctx, zkeyBytes) -> handle (sync: done once per key) ; groth16Prove(ctx, handle, witnessSection, r, s) -> Promise<Buffer(8*n8q)>
Napi::Value Groth16Load(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); auto z = info[1].As<Napi::Uint8Array>(); uint64_t h = 0;
  if (sb_groth16_load(c, z.Data(), z.ByteLength(), &h)) { Napi::Error::New(info.Env(), sb_last_error(c)).ThrowAsJavaScriptException(); return info.Env().Undefined(); }
  return Napi::Number::New(info.Env(), (double)h);
}
Napi::Value Groth16Prove(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); uint64_t h = (uint64_t)info[1].As<Napi::Number>().Int64Value();
  auto w = info[2].As<Napi::Uint8Array>(); auto r = info[3].As<Napi::Uint8Array>(); auto s = info[4].As<Napi::Uint8Array>();
  size_t n8q = info[5].As<Napi::Number>().Uint32Value();
  size_t nw = w.ByteLength() / 32; const uint8_t *pw = w.Data(), *pr = r.Data(), *ps = s.Data();
  return Queue(info.Env(), c, 8 * n8q, [=](std::vector<uint8_t>& out) { return sb_groth16_prove(c, h, pw, nw, pr, ps, out.data()); }, {w, r, s});
}

// groth16LoadFile(ctx, path) -> handle: the zkey is streamed from disk through pinned buffers (sb_groth16_load_file), never
// materialised in the JS heap; groth16ProveWtns(ctx, handle, wtnsFileBytes, r, s, n8q) -> Promise<Buffer(8*n8q)>
Napi::Value Groth16LoadFile(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); std::string path = info[1].As<Napi::String>().Utf8Value(); uint64_t h = 0;
  if (sb_groth16_load_file(c, path.c_str(), &h)) { Napi::Error::New(info.Env(), sb_last_error(c)).ThrowAsJavaScriptException(); return info.Env().Undefined(); }
  return Napi::Number::New(info.Env(), (double)h);
}
Napi::Value Groth16ProveWtns(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); uint64_t h = (uint64_t)info[1].As<Napi::Number>().Int64Value();
  auto w = info[2].As<Napi::Uint8Array>(); auto r = info[3].As<Napi::Uint8Array>(); auto s = info[4].As<Napi::Uint8Array>();
  size_t n8q = info[5].As<Napi::Number>().Uint32Value();
  size_t wl = w.ByteLength(); const uint8_t *pw = w.Data(), *pr = r.Data(), *ps = s.Data();
  return Queue(info.Env(), c, 8 * n8q, [=](std::vector<uint8_t>& out) { return sb_groth16_prove_wtns(c, h, pw, wl, pr, ps, out.data()); }, {w, r, s});
}
Napi::Value Groth16Info(const Napi::CallbackInfo& info) {
  uint32_t nv = 0, np = 0, ds = 0;
  sb_groth16_info(ctx_of(info[0]), (uint64_t)info[1].As<Napi::Number>().Int64Value(), &nv, &np, &ds);
  Napi::Object o = Napi::Object::New(info.Env());
  o.Set("nVars", nv); o.Set("nPublic", np); o.Set("domainSize", ds);
  return o;
}
Napi::Value Groth16Release(const Napi::CallbackInfo& info) {
  sb_groth16_release(ctx_of(info[0]), (uint64_t)info[1].As<Napi::Number>().Int64Value());
  return info.Env().Undefined();
}

// plonkLoad / fflonkLoad(ctx, zkeyBytes) -> handle ; plonkProve / fflonkProve(ctx, handle, witnessSection, blinders) -> Promise<Buffer>
// (src/plonk_prove.js:47, src/fflonk_prove.js:51; blinders = 11 resp. 9 Fr.random() elements concatenated)
template <int (*LOAD)(sb_ctx*, const uint8_t*, uint64_t, uint64_t*)>
Napi::Value KeyLoad(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); auto z = info[1].As<Napi::Uint8Array>(); uint64_t h = 0;
  if (LOAD(c, z.Data(), z.ByteLength(), &h)) { Napi::Error::New(info.Env(), sb_last_error(c)).ThrowAsJavaScriptException(); return info.Env().Undefined(); }
  return Napi::Number::New(info.Env(), (double)h);
}
template <int (*PROVE)(sb_ctx*, uint64_t, const uint8_t*, uint64_t, const uint8_t*, uint8_t*), uint32_t (*BYTES)(sb_ctx*)>
Napi::Value KeyProve(const Napi::CallbackInfo& info) {
  sb_ctx* c = ctx_of(info[0]); uint64_t h = (uint64_t)info[1].As<Napi::Number>().Int64Value();
  auto w = info[2].As<Napi::Uint8Array>(); auto b = info[3].As<Napi::Uint8Array>();
  size_t nw = w.ByteLength() / 32; const uint8_t *pw = w.Data(), *pb = b.Data();
  return Queue(info.Env(), c, BYTES(c), [=](std::vector<uint8_t>& out) { return PROVE(c, h, pw, nw, pb, out.data()); }, {w, b});
}

Napi::Object Init(Napi::Env env, Napi::Object exports) {
  exports.Set("createContext", Napi::Function::New(env, Create));
  exports.Set("multiExpAffine", Napi::Function::New(env, MultiExpAffine));
  exports.Set("nttFr", Napi::Function::New(env, NttFr));
  exports.Set("frBatchApplyKey", Napi::Function::New(env, FrBatchApplyKey));
  exports.Set("frConvert", Napi::Function::New(env, FrConvert));
  exports.Set("qapJoinAbc", Napi::Function::New(env, QapJoinAbc));
  exports.Set("groupFft", Napi::Function::New(env, GroupFft));
  exports.Set("groupApplyKey", Napi::Function::New(env, GroupApplyKey));
  exports.Set("groth16Load", Napi::Function::New(env, Groth16Load));
  exports.Set("groth16Prove", Napi::Function::New(env, Groth16Prove));
  exports.Set("groth16LoadFile", Napi::Function::New(env, Groth16LoadFile));
  exports.Set("groth16ProveWtns", Napi::Function::New(env, Groth16ProveWtns));
  exports.Set("groth16Info", Napi::Function::New(env, Groth16Info));
  exports.Set("groth16Release", Napi::Function::New(env, Groth16Release));
  exports.Set("plonkLoad", Napi::Function::New(env, KeyLoad<sb_plonk_load>));
  exports.Set("plonkProve", Napi::Function::New(env, KeyProve<sb_plonk_prove, sb_plonk_proof_bytes>));
  exports.Set("fflonkLoad", Napi::Function::New(env, KeyLoad<sb_fflonk_load>));
  exports.Set("fflonkProve", Napi::Function::New(env, KeyProve<sb_fflonk_prove, sb_fflonk_proof_bytes>));
  return exports;
}

}  // namespace

NODE_API_MODULE(snarkb200_napi, Init)
