"""The FP16 transformer flow's FFN convolutions at the shape the engine runs them.  The flow's FFN kernel size is flow_kernel_size = 5
(reference models.py:905, 917; conv_from takes K from the weights), while the f16.ffn1 / f16.ffn2 families of kernel_cases.py run K = 3;
these families are the same calls at K = 5, with the same case scheme (edge lengths, ragged batches, forced dispatch)."""
from unittest import mock

import kernel_cases as KC

FAMILIES = {
    "f16.ffn1_k5": dict(KC.FAMILIES["f16.ffn1"], K=5),
    "f16.ffn2_k5": dict(KC.FAMILIES["f16.ffn2"], K=5),
}


def conv_cases():
    """(id, family name, B, T, lens, num_sms, expected plan or None), as kernel_cases.conv_cases()"""
    out = []
    for name, f in FAMILIES.items():
        for T in KC.EDGE_T:
            out.append((f"{name}-T{T}-B1", name, 1, T, [T], KC.H100_SMS, None))
        for T in (300, 1000):
            out.append((f"{name}-T{T}-B3", name, 3, T, KC._ragged(T), KC.H100_SMS, None))
        out.append((f"{name}-T1023-B1", name, 1, 1023, [1023], KC.H100_SMS, dict(kind="one-tile")))  # the config-2 flow
        out.append((f"{name}-T300-B3-sms{KC.BIG_SMS}", name, 3, 300, KC._ragged(300), KC.BIG_SMS, dict(kind="one-tile")))
        out.append((f"{name}-T300-B3-sms{KC.SMALL_SMS}", name, 3, 300, KC._ragged(300), KC.SMALL_SMS, dict(kind=f["small"])))
    return out


def family_args(name, B, T, lens, num_sms):
    """kernel_cases.family_args of one of these families"""
    with mock.patch.dict(KC.FAMILIES, {name: FAMILIES[name]}):
        return KC.family_args(name, B, T, lens, num_sms)
