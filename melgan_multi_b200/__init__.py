"""melgan_multi_b200: H100-native (sm_90a) engine for the MelGAN hot path of diver-j/melgan-multi.

``melgan_multi_b200.models`` is the drop-in for the reference's ``models`` module; ``engine`` binds
the C ABI of libmelgan_b200.so (include/melgan_b200.h); ``synth`` makes the seeded weights/inputs
used by tests and benchmarks; ``build`` compiles the library in-tree for sm_90a.
"""
__all__ = ["models", "engine", "synth", "build"]
