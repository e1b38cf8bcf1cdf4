"""Hindsight Experience Replay (baselines/her/) on the sm_90a kernels of csrc/her.cu."""
