"""mmssl_b200 -- the MMSSL training step (HKUDS/MMSSL) on H100, hand-written CUDA behind a C ABI.

  Models          drop-in for the reference's Models.py (MMSSL as one autograd node, Discriminator)
  functional      autograd wrappers: SpMMFunction, bpr_loss, batched_contrastive_loss, feat_reg_loss
  engine          forward / backward schedule of the hot path over the library kernels
  hotstep         fused hot step (loss kernels + backward + AdamW), CUDA-graph captured
  gan, gan_ops    the GAN side without autograd (Discriminator sweeps, gradient penalty, u_sim)
  fullstep        the whole training iteration of main.py:333-434 on the device
  trainer         mirror of the reference's Trainer life cycle (train / test)
  evaluate        fused ranking + metrics (utility/batch_test.py)
  sampler         Data.sample on the device
  dataset         reader of the reference's dataset directory, memory-mapped per-rank shards
  parallel        data-parallel bucket / fused multimem optimiser, row-sharded propagation, symmetric tables
  rowshard_step   the whole hot step under the row-sharded scheme (NCCL or multicast exchange)
  graph, ops, _lib   prepared sparse operands, tensor-level wrappers, ctypes binding of libmmssl_b200.so
  build           nvcc build of the library (sm_90a)

Nothing is imported here: `import mmssl_b200` stays cheap, every sub-module loads the library on first use and refuses to run
without it and an H100 (no CPU or eager-PyTorch fallback)."""
