// snarkb200.mjs — overrides the bulk methods of snarkjs' curve singleton with the CUDA backend.
// Usage:  import { useB200 } from "./snarkb200.mjs";  await useB200("bn128");  await snarkjs.groth16.prove(zkey, wtns);
// Not runnable in this repository's image (no Node.js); see INTEGRATION.md for the line-by-line rationale.
import { createRequire } from "module";
import * as snarkjs from "snarkjs";
const addon = createRequire(import.meta.url)("./build/Release/snarkb200_napi.node");

const flatten = (b) => (b instanceof Uint8Array ? b : Buffer.concat(b.buffers));          // BigBuffer (ffjavascript 12692-12778)

export async function useB200(curveName = "bn128", device = 0) {
  const curve = await snarkjs.curves.getCurveFromName(curveName);                           // the singleton snarkjs itself gets (src/curves.js:36-53)
  const ctx = addon.createContext(curveName === "bn128" ? 0 : 1, device);
  const n8q = curve.F1.n8;
  for (const [G, gid] of [[curve.G1, 1], [curve.G2, 2]]) {
    G.multiExpAffine = async (buffBases, buffScalars) => {
      const bases = flatten(buffBases), scalars = flatten(buffScalars);
      const n = Math.floor(bases.byteLength / (G.F.n8 * 2));
      if (n == 0) return G.zero;
      if (Math.floor(scalars.byteLength / n) * n != scalars.byteLength) throw new Error("Scalar size does not match");
      return new Uint8Array(await addon.multiExpAffine(ctx, gid, bases, scalars, n8q));
    };
  }
  const Fr = curve.Fr;
  // G.fft / G.ifft / G.lagrangeEvaluations / G.batchApplyKey (build/snarkjs.js:15101-15176, 14268-14385): every butterfly is a
  // scalar multiplication on the GPU.  Array inputs (one Uint8Array per point) come back as arrays, like Fr.fft below.
  for (const [G, gid] of [[curve.G1, 1], [curve.G2, 2]]) {
    const size = (t) => G.F.n8 * ((t || "affine") == "jacobian" ? 3 : 2);
    const gfft = (inverse) => async (buff, inType, outType) => {
      const isArray = Array.isArray(buff);
      const b = isArray ? Buffer.concat(buff) : flatten(buff);
      const n = b.byteLength / size(inType);
      if (!Number.isInteger(Math.log2(n))) throw new Error("fft must be multiple of 2");
      const out = new Uint8Array(await addon.groupFft(ctx, gid, b, +(inType == "jacobian"), inverse, +(outType == "jacobian"), n8q));
      const so = size(outType);
      return isArray ? Array.from({ length: n }, (_, i) => out.slice(i * so, (i + 1) * so)) : out;
    };
    G.fft = gfft(0);
    G.ifft = gfft(1);
    G.lagrangeEvaluations = async (buff, inType, outType) => {
      const b = flatten(buff), bits = Math.log2(b.byteLength / size(inType));
      if (!Number.isInteger(bits)) throw new Error("lagrangeEvaluations invalid Input size");
      if (bits > Fr.s + 1) throw new Error("lagrangeEvaluations input too big");
      return G.ifft(b, inType, outType);                                                     // Fr.s + 1 is refused by the library
    };
    G.batchApplyKey = async (buff, first, inc, inType, outType) =>
      new Uint8Array(await addon.groupApplyKey(ctx, gid, flatten(buff), Fr.e(first), Fr.e(inc), +(inType == "jacobian"), +(outType == "jacobian"), n8q));
  }
  const fft = (inverse) => async (buff) => {
    const isArray = Array.isArray(buff);
    const b = isArray ? Buffer.concat(buff) : flatten(buff);
    const n = b.byteLength / Fr.n8;
    if (!Number.isInteger(Math.log2(n))) throw new Error("fft must be multiple of 2");
    const out = new Uint8Array(await addon.nttFr(ctx, b, inverse));
    return isArray ? Array.from({ length: n }, (_, i) => out.slice(i * Fr.n8, (i + 1) * Fr.n8)) : out;
  };
  Fr.fft = fft(0);
  Fr.ifft = fft(1);
  Fr.batchApplyKey = async (buff, first, inc) => new Uint8Array(await addon.frBatchApplyKey(ctx, flatten(buff), Fr.e(first), Fr.e(inc)));
  Fr.batchToMontgomery = async (buff) => new Uint8Array(await addon.frConvert(ctx, flatten(buff), 1));
  Fr.batchFromMontgomery = async (buff) => new Uint8Array(await addon.frConvert(ctx, flatten(buff), 0));
  const queueAction = curve.tm.queueAction.bind(curve.tm);
  curve.tm.queueAction = async (task) => {                                                 // joinABC's raw tasks (src/groth16_prove.js:338-355)
    const call = task.find((t) => t.cmd == "CALL");
    if (call && call.fnName == "qap_joinABC") {
      const [a, b, c] = task.filter((t) => t.cmd == "ALLOCSET").map((t) => t.buff);
      return [new Uint8Array(await addon.qapJoinAbc(ctx, a, b, c))];
    }
    return queueAction(task);
  };
  // Fused route: groth16Prove(zkeyFileName, witnessFileName) with the signature and result of src/groth16_prove.js:28-144.
  // The key goes to HBM once per file (cache keyed by path + size + mtime: the device copy and its window tables are
  // reused by every later proof); a proof is then ONE addon call (witness in, 3 affine points out) instead of ~25 bulk
  // calls with host round trips.  snarkjs' own `groth16.prove` is an ES-module export and cannot be reassigned, so callers
  // switch by importing this function (or by passing `options.backend = b200` to a patched cli.js, INTEGRATION.md).
  const keys = new Map();
  const groth16Prove = async (zkeyFileName, witnessFileName, logger) => {
    const fs = await import("fs");
    const st = fs.statSync(zkeyFileName);
    const tag = `${zkeyFileName}:${st.size}:${st.mtimeMs}`;
    if (!keys.has(tag)) keys.set(tag, addon.groth16LoadFile(ctx, zkeyFileName));
    const wtns = fs.readFileSync(witnessFileName);
    const r = curve.Fr.random(), s = curve.Fr.random();                                     // src/groth16_prove.js:103-104
    const raw = new Uint8Array(await addon.groth16ProveWtns(ctx, keys.get(tag), wtns, r, s, n8q));
    const G1 = curve.G1, G2 = curve.G2, sG1 = 2 * n8q, sG2 = 4 * n8q;
    const proof = { pi_a: G1.toObject(raw.slice(0, sG1)), pi_b: G2.toObject(raw.slice(sG1, sG1 + sG2)), pi_c: G1.toObject(raw.slice(sG1 + sG2)),
                    protocol: "groth16", curve: curve.name };                                // :130-141
    // public signals: witness values 1..nPublic (:134-139); nPublic comes from the zkey header
    const { nPublic } = addon.groth16Info ? addon.groth16Info(ctx, keys.get(tag)) : { nPublic: 0 };
    const n8r = curve.Fr.n8;
    const sec2 = locateWtnsSection2(wtns);
    const publicSignals = [];
    for (let i = 1; i <= nPublic; i++) publicSignals.push(BigInt("0x" + Buffer.from(wtns.subarray(sec2 + i * n8r, sec2 + (i + 1) * n8r)).reverse().toString("hex")));
    return snarkjs.utils ? { proof: snarkjs.utils.stringifyBigInts(proof), publicSignals: snarkjs.utils.stringifyBigInts(publicSignals) } : { proof, publicSignals };
  };
  return { curve, ctx, addon, groth16Prove };
}

// offset of section 2's payload in a .wtns image (binfile container: "wtns" u32 version u32 nSections, then (u32 id, u64 len, payload)*)
function locateWtnsSection2(buf) {
  let pos = 12;
  const n = buf.readUInt32LE(8);
  for (let i = 0; i < n; i++) {
    const id = buf.readUInt32LE(pos), len = Number(buf.readBigUInt64LE(pos + 4));
    if (id == 2) return pos + 12;
    pos += 12 + len;
  }
  throw new Error("wtns: section 2 missing");
}
