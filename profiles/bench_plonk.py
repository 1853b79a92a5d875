"""PLONK / fflonk timing by domain size (planning data, not the headline bench): synthetic satisfiable circuits built by
oracle/plonk.py's setup on unstructured points, proofs through sb_plonk_prove with the witness in host memory.
Prints one JSON line per size as soon as it is measured.
usage: python profiles/bench_plonk.py [plonk|fflonk] [budget_seconds] [log2 sizes ...]"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("OMP_NUM_THREADS", "8")   # the CPU-side key setup is many small oracle calls: wide OpenMP teams only add latency
T0 = time.time()
import numpy as np                      # noqa: E402
import snarkjs_b200                     # noqa: E402
from oracle import oracle as orc        # noqa: E402
from oracle import plonk as op          # noqa: E402

from oracle import fflonk as off       # noqa: E402

argv = sys.argv[1:]
proto = argv.pop(0) if argv and argv[0] in ("plonk", "fflonk") else "plonk"
budget = float(argv[0]) if argv else 45.0
sizes = [int(a) for a in argv[1:]] or [14, 16, 18]
mod = snarkjs_b200.plonk if proto == "plonk" else snarkjs_b200.fflonk
n_blinders = 11 if proto == "plonk" else 9
curve = snarkjs_b200.getCurveFromName("bn128")
ci = orc.CURVES[orc.BN254]
bl = b"".join(ci.fr_to_mont(7 + i) for i in range(n_blinders))
est = {14: 6, 16: 14, 18: 45, 20: 200}
for lg in sizes:
    if time.time() - T0 + est.get(lg, 10) > budget:
        print("skip 2^%d: out of time budget" % lg)
        continue
    t = time.time()
    gates, adds, n_vars, n_pub, wit = op.chain_gates((1 << lg) - 6)
    setup = op.plonk_setup_synth if proto == "plonk" else off.fflonk_setup_synth
    zkey = setup(gates, adds, n_vars, n_pub, tau=4242, structured=False)
    t_setup = time.time() - t
    W = np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in wit), np.uint8)
    t = time.time()
    pk = mod.ProvingKey(zkey, curve)
    t_load = time.time() - t
    del zkey
    first = pk.prove_raw(W, bl)
    ms, dev, rounds = [], [], []
    l0 = curve.launch_count()
    reps = 5 if lg <= 16 else 3
    for _ in range(reps):
        t = time.perf_counter()
        raw = pk.prove_raw(W, bl)
        ms.append((time.perf_counter() - t) * 1e3)
        dev.append(curve.last_ms(0))
        rounds.append([curve.last_ms(i) for i in range(1, 6)])
    launches = (curve.launch_count() - l0) // reps
    assert raw == first
    line = {"what": proto + "_prove", "curve": "bn128", "log2_domain": lg, "n_public": n_pub, "n_additions": len(adds),
            "ms_e2e_median": round(float(np.median(ms)), 3), "ms_min": round(min(ms), 3), "proofs_per_s": round(1e3 / float(np.median(ms)), 2),
            "ms_flow_device_clock": round(float(np.median(dev)), 3), "launches_per_proof": int(launches),
            "ms_rounds_1_to_5": [round(float(x), 3) for x in np.median(np.array(rounds), axis=0)],
            "key_load_s": round(t_load, 2), "cpu_setup_s": round(t_setup, 1), "witness_bytes": int(W.size)}
    print(json.dumps(line), flush=True)
    pk.release()
curve.terminate()
