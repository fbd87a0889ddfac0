"""codebase_b200 -- H100 (sm_90a) hot path of marlbase (marl-book/codebase): the LBF env-step loop,
episode replay / on-policy storage and the IDQN / VDN / IA2C learner updates as hand-written CUDA behind a C ABI,
mirrored on the host side by the reference's own Python plugin surface."""
__version__ = "0.1.0"
