"""H100-native Multi-HMR inference path (sm_90a CUDA kernels behind the reference's Model.forward API).

The directory is named after the project (`multi-hmr_b200`); import it as `multihmr_b200`.
"""
