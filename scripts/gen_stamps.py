"""Regenerate data/_stamps.py from the reference PNG assets (needs cv2 + the PNGs).

Usage: python scripts/gen_stamps.py REFERENCE_ROOT
Mirrors the array the reference computes at src/utils.py:232-242 (bitwise_not -> cubic resize to 28x28).
"""
import sys
import cv2
import numpy as np

if len(sys.argv) != 2:
    sys.exit(__doc__)
root = sys.argv[1]
for key, name in [("copyright", "watermark"), ("apple", "apple")]:
    t = cv2.imread(f"{root}/{name}.png", cv2.IMREAD_GRAYSCALE)
    t = cv2.resize(cv2.bitwise_not(t), dsize=(28, 28), interpolation=cv2.INTER_CUBIC)
    print(f"{key.upper()}_28 =", [(int(r), int(c), int(t[r, c])) for r, c in np.argwhere(t > 0)])
