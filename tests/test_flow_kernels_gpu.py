"""Kernel-level parity of the FP16 flow's FFN convolutions at K = 5 on an H100: the checks of test_kernels_gpu.test_tc_conv1d (float64
reference with the kernel's operand rounding, untouched channels, guard regions, error flag, bitwise repeatable) on the families of
flow_kernel_cases.py.  Run: pytest -m gpu tests/test_flow_kernels_gpu.py -v -s"""
import pytest

import flow_kernel_cases as FC
import kernel_cases as KC
import test_kernels_gpu as TK

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cid,fam,B,T,lens,sms,expect", FC.conv_cases(), ids=[c[0] for c in FC.conv_cases()])
def test_tc_conv1d_flow_ffn_k5(monkeypatch, cid, fam, B, T, lens, sms, expect):
    monkeypatch.setitem(KC.FAMILIES, fam, FC.FAMILIES[fam])
    TK.test_tc_conv1d(cid, fam, B, T, lens, sms, expect)
