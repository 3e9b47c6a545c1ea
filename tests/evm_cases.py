"""Configurations of the LNES='EVM' tests (tests/golden/make_golden_evm.py records them from the reference): settings 1-3 on three bins."""
from harness import ITEM_SET

EVM_BINS = {"10": (10, 10, 10), "14x12": (14, 12, 10), "20": (20, 20, 20)}
EVM_CASES = {"s%d_%s" % (s, b): dict(setting=s, container=c, items=ITEM_SET, nb=80, nl=50, steps=70, seed=5, env=0, lnes="EVM")
             for s in (1, 2, 3) for b, c in EVM_BINS.items()}
