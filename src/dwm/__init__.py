"""Drop-in mirror of the `dwm` package surface that OpenDWM's CTSD denoising hot path
needs (config factory, DiT model, per-frame schedulers, ctsd pipelines), executing on
the H100-native kernels of `opendwm_b200` through its C ABI."""
