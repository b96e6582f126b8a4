"""ORACLE SUPPORT (test infrastructure, NOT product code): the stereo Frame constructor (src/Frame.cc:101-197) restated on the CPU for the
tests of the stereo path: the two ORBextractor calls on the rectified left and right images, then Frame::ComputeStereoMatches
(oracle.stereo_matches), as a frame builder whose output oracle.chain.oracle_chain2 takes."""
import numpy as np

import oracle


def stereo_frame(ex_left: "oracle.Extractor", ex_right: "oracle.Extractor", left: np.ndarray, right: np.ndarray, mb, mbf) -> dict:
    """mvKeys / mDescriptors of the left image, mvDepth / mvuRight from ComputeStereoMatches (mvKeysUn == mvKeys: rectified images)
    -> dict(k, d, depth, ur).  Each extractor keeps the pyramid of its image, which the SAD refinement reads."""
    k, d, _ = ex_left(left)
    kr, dr, _ = ex_right(right)
    dep, ur = oracle.stereo_matches(k, d, kr, dr, ex_left, ex_right, np.float32(mb), np.float32(mbf))
    return dict(k=k, d=d, depth=dep, ur=ur)
