"""distributed_plonk_b200 - H100-native (sm_90a) MSM + NTT hot path of MengLing-L/distributed_plonk.

  csrc/         hand-written CUDA kernels + the C ABI (include/dplonk.h)
  _binding.py   ctypes view of the C ABI
  worker.py     host-side mirror of the reference's PlonkSlave / PlonkPeer RPC surface (worker.rs)
  dispatcher.py host-side mirror of the dispatcher's Prover::fft / commit_polynomial (dispatcher2.rs)
  parallel.py   one-process-per-GPU plumbing (torch.distributed all-to-all for the 2-D NTT exchange)
"""
from ._binding import Context, DpError, FftWorkload  # noqa: F401
from ._lib import ExtensionMissing, library_path, load  # noqa: F401

__all__ = ["Context", "DpError", "FftWorkload", "ExtensionMissing", "library_path", "load"]
