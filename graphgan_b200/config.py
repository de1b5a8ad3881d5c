"""Run-time configuration: the reference's ``config`` surface, name for name and default for default.

The reference keeps its hyper-parameters as attributes of a flat module that every layer reads at CALL
time (``config.<name>``; reference src/GraphGAN/config.py:1-41), so callers and tests can patch
them.  This module is that flat module: the same names with the same values (they are the API), followed
by the knobs of this implementation, whose defaults leave the reference behaviour unchanged.
``src/GraphGAN/config.py`` aliases this module so ``import config`` keeps working from that directory.
"""

# ---- the two models, in the order of the embedding / result files (reference config.py:1)
modes = ["gen", "dis"]

# ---- optimisation schedule (reference config.py:4-16)
n_epochs = 20                       # outer loops
n_epochs_dis = 30                   # discriminator inner loops per outer loop
n_epochs_gen = 30                   # generator inner loops per outer loop
dis_interval = n_epochs_dis         # resample discriminator data every this many inner loops
gen_interval = n_epochs_gen         # same for the generator
batch_size_dis = 64                 # pairs per discriminator step (any size; above 1024 the gradient runs multi-CTA)
batch_size_gen = 64                 # pairs per generator step (likewise, also data parallel under torchrun)
lr_dis = 1e-3                       # Adam learning rates
lr_gen = 1e-3
lambda_dis = 1e-5                   # l2 weights of the two losses
lambda_gen = 1e-5
n_sample_gen = 20                   # walks per root in a generator pass
update_ratio = 1                    # fraction of roots resampled per pass
window_size = 2                     # skip-gram window of get_node_pairs_from_path

# ---- model shape and checkpointing (reference config.py:19-25)
n_emb = 50
load_model = False
save_steps = 10
multi_processing = False            # accepted for compatibility: trees are built on the GPU

# ---- task, dataset and the nine path strings (reference config.py:28-41), relative to src/GraphGAN
app = "link_prediction"
dataset = "CA-GrQc"
_data = "../../data/" + app + "/" + dataset
_results = "../../results/" + app + "/" + dataset
train_filename = _data + "_train.txt"
test_filename = _data + "_test.txt"
test_neg_filename = _data + "_test_neg.txt"
pretrain_emb_filename_d = "../../pre_train/" + app + "/" + dataset + "_pre_train.emb"
pretrain_emb_filename_g = pretrain_emb_filename_d
emb_filenames = [_results + "_gen_.emb", _results + "_dis_.emb"]
result_filename = _results + ".txt"
cache_filename = "../../cache/" + dataset + ".pkl"      # unused here: trees are rebuilt on the GPU
model_log = "../../log/"

# ---- additions of this implementation (not in the reference)
device = "cuda:0"                   # one process per GPU; LOCAL_RANK overrides the index under torchrun
seed = 0                            # Philox key of the walk sampler and seed of the batch shuffles
root_batch = 4096                   # roots whose BFS tree rows are resident at once (nnz / 8 bytes each)
tree_cache_bytes = 8 << 30          # keep ALL trees resident (like the reference's cache) below this size
max_path_len = 64                   # row stride of recorded generator paths; a longer walk is an error
text_embeddings = True              # the reference's text dump (graph_gan.py:293-306); turn off at N >= 1e5 (minutes per epoch)
binary_embeddings = False           # also dump <emb_filename>.f32 (header + [N, n_emb] fp32, row-major) every epoch
device_eval = True                  # link-prediction check on the GPU (io/evaluation text round trip skipped)
value_roots = 0                     # > 0: evaluation also writes "value:<V> pos:<..> neg:<..> roots:<n>", the exact game value
value_grad = False                 # with value_roots > 0: the value line also ends in " gnorm:<|grad_G mean V|_2>", exact
                                    # (DESIGN.md section 5.2) averaged over this many seeded roots (rank 0's shard under torchrun)
value_grad_d = False               # with value_roots > 0: the value line ends in " dnorm:<|grad_D mean V|_2>", exact (section 5.4)
value_gcos = False                 # with value_roots > 0: the value line ends in " gcos:<cos>", the cosine between the exact
                                    # expectation of the reference's G step and grad_G V (DESIGN.md section 5.6)
value_dcos = False                 # with value_roots > 0: the value line ends in " dcos:<cos>" (after gcos), the cosine
                                    # between the exact expectation of the reference's D step and grad_D V (section 5.7)
value_jsd = False                  # with value_roots > 0: the value line ends in " jsd:<mean JSD> hit:<mean hit>" (after
                                    # dcos): G's exact Jensen-Shannon divergence from the data and its mass on the true
                                    # neighbours, from the top two levels of each tree (DESIGN.md section 5.8)
value_gsnr = False                 # with value_roots > 0: the value line ends in " gsnr:<n |M|^2 / sum var_c>" (after jsd):
                                    # the signal-to-noise ratio of one sampled G pass of n = n_sample_gen walks per root,
                                    # exact (DESIGN.md section 5.9)
exact_roots = 0                     # > 0: train() plays the exact game on this many seeded roots (DESIGN.md section 5.5):
                                    # each D / G step is an Adam step on the exact gradient of the mean V; no walks are
                                    # sampled.  Single process only.  0: the reference's sampled training
