"""Selective-scan cases at 32 and 64 states, shared by oracle/gen_dstate_golden.py and the tests that read its golden vectors."""

DSTATE_CASES = [
    # name, seed, batch, dim, L, N, G, trained_like, has_D, has_z, has_bias, softplus
    ("dstate32_L97", 20, 2, 4, 97, 32, 1, False, True, True, True, True),
    ("dstate32_L600_g2_plain", 21, 1, 4, 600, 32, 2, False, False, False, False, False),
    ("dstate64_L97_g2", 22, 2, 4, 97, 64, 2, False, True, True, True, True),
    ("dstate64_L600_plain", 23, 1, 4, 600, 64, 1, False, False, False, False, False),
    ("dstate64_trained_L300_d40", 24, 1, 40, 300, 64, 1, True, True, True, True, True),
]
