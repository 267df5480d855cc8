"""
dragonfly_b200 -- the H100 (sm_90a) GP-BO inner loop behind Dragonfly's Kernel / GP /
gpb_acquisitions surfaces.  See DESIGN.md.  Importing the package does not touch the GPU; the first
device call loads libdfb200.so and fails loudly if it (or a CUDA device) is missing.
"""
__version__ = '0.1.0'
