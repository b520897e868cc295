"""beat_this_b200 -- the CPJKU/beat_this Audio -> Beats inference path as hand-written
sm_90a (H100) CUDA behind the reference's ``beat_this.inference`` API."""
__version__ = "0.1.0"
