"""snarkjs_b200 — H100 (sm_90a) backend for snarkjs' bulk curve operations (MSM, NTT) and a fused Groth16 prover.

Package layout: csrc/ (CUDA kernels + C ABI -> libsnarkb200.so), curve.py (mirror of the ffjavascript curve
object's bulk methods), groth16.py (mirror of src/groth16_prove.js), plonk.py (mirror of src/plonk_prove.js), fflonk.py (mirror of src/fflonk_prove.js)."""
from .curve import Curve, SbError, getCurveFromName, getCurveFromQ, getCurveFromR  # noqa: F401
from . import groth16  # noqa: F401
from . import plonk  # noqa: F401
from . import fflonk  # noqa: F401
