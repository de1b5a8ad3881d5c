"""Flat drop-in aliases of graphgan_b200.{config,generator,discriminator,graph_gan} under the reference's directory
layout (INTEGRATION.md section 2): `import config`, `import generator`, ... from this directory resolve to the CUDA build."""
