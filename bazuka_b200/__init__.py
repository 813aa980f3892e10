"""bazuka_b200 — H100-native kernels for Bazuka's MPN Groth16 proving path.

Host-side mirror of the reference's interfaces for this path, over libbzk's C ABI:

  reference (Rust)                                         here
  ----------------------------------------------------     ------------------------------------
  zk::ZkScalar                      src/zk/mod.rs:202      numpy uint64[4] Montgomery image (`fr`)
  zk::poseidon::poseidon(vals)      poseidon/mod.rs:81     Context.poseidon(inputs)
  zk::ZkHasher::hash                src/zk/mod.rs:152      Context.poseidon (batched)
  bellman EvaluationDomain::{fft,ifft,coset_fft,icoset_fft}   Context.ntt(a, op)
  bellman multiexp (G1 / G2)                                Context.msm_g1 / msm_g2, G1Bases/G2Bases
  groth16 wire tuples               groth16/mod.rs:19-38   uint8[104] / uint8[200] images

Device memory and streams come from torch (plumbing only); every computation is a libbzk kernel.
"""
from ._lib import BzkError, load, SO_PATH  # noqa: F401
from .api import Context, G1Bases, G2Bases, NTT_FFT, NTT_IFFT, NTT_COSET_FFT, NTT_ICOSET_FFT  # noqa: F401

__all__ = ["Context", "G1Bases", "G2Bases", "BzkError", "load",
           "NTT_FFT", "NTT_IFFT", "NTT_COSET_FFT", "NTT_ICOSET_FFT"]
