"""Writes tests/golden/sift_000012.npz from a checkout of the reference project (data files only, no source):

    python tests/golden/make_sift_golden.py <reference checkout>

Inputs: src/test/resources/images/000012.jpg and images/feats128.csv, the 128 x 64990 descriptors SIFTExtractor(scaleStep = 0)
gives for that image after PixelScaler and GrayScaler (one descriptor per column, integers in [0, 255]; no reference test reads
the csv, DESIGN.md section 18 records how it was identified).  To keep the fixture small it holds
  rgb    the image decoded once with PIL to 8-bit RGB (333 x 500 x 3);
  zero   for every one of the 64990 keypoints, whether its descriptor is all zero (the contrast threshold);
  cols   every 32nd keypoint, 0, 32, ...;
  feats  the full descriptors of those keypoints, uint8 128 x len(cols), columns as in the csv."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
STRIDE = 32


def main(ref_root: str) -> None:
    from PIL import Image
    images = os.path.join(ref_root, "src", "test", "resources", "images")
    rgb = np.array(Image.open(os.path.join(images, "000012.jpg")).convert("RGB"), dtype=np.uint8)
    feats = np.loadtxt(os.path.join(images, "feats128.csv"), delimiter=",", dtype=np.int64)
    assert feats.shape == (128, 64990) and feats.min() >= 0 and feats.max() <= 255
    cols = np.arange(0, feats.shape[1], STRIDE, dtype=np.int32)
    np.savez_compressed(os.path.join(HERE, "sift_000012.npz"), rgb=rgb, zero=(feats == 0).all(0), cols=cols,
                        feats=feats[:, cols].astype(np.uint8))
    print("wrote", os.path.join(HERE, "sift_000012.npz"))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
