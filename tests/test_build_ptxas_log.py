"""build.py rejects a ptxas log that reports serialised wgmma (C7510)."""
from audiolm_pytorch_b200 import build


def test_c7510_is_reported_per_kernel():
    log = (
        "ptxas info    : (C7510) Potential Performance Loss: wgmma.mma_async instructions are serialized due to wgmma "
        "pipeline crossing function boundary at a function call in the function '_ZN3alm6kernelEv'\n"
        "ptxas info    : Used 168 registers, used 1 barriers\n"
    )
    assert build._wgmma_serialised(log) == ["_ZN3alm6kernelEv"]


def test_clean_log_passes():
    log = "ptxas info    : Compiling entry function '_ZN3alm6kernelEv' for 'sm_90a'\nptxas info    : Used 253 registers\n"
    assert build._wgmma_serialised(log) == []
