"""graphgan_b200 -- H100 (sm_90a) implementation of GraphGAN's scoring-and-sampling hot path.

Scope (SURVEY.md section 8): the graph-softmax walk sampler, BFS-tree construction, pairwise
discriminator/generator scoring, reward, sparse gradients and the TF1-style Adam update, behind
the reference's ``Generator`` / ``Discriminator`` / ``config`` Python surface.  All computation
lives in libgraphgan_b200.so (hand-written CUDA, C ABI in include/graphgan_b200.h); torch is
used for device memory, streams and torch.distributed only.  There is no CPU fallback.
"""
__version__ = "0.1.0"
