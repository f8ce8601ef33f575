"""uisrnn_b200 -- H100-native (sm_90a) implementation of UIS-RNN's predict() hot path behind
the reference's Python API.  `import uisrnn` (the alias package at the repo root) gives the
drop-in surface of google/uis-rnn; this package holds the host-side mirror and the native code.
"""
__version__ = '0.1.0'
