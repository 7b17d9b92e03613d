"""TEST INFRASTRUCTURE: the CPU oracle (oracle/monodetr_torch.py, tests/oracle_dab.py) at the reference's other transformer
sizes -- cfg["enc_layers"] / cfg["dec_layers"] 1 to 6, cfg["num_queries"] up to 300, cfg["dim_feedforward"] and
cfg["aux_loss"].  The oracle already takes the layer counts, the query count and the FFN width from its cfg; what this module adds
is the variant table, the cfg of each variant, and `aux_loss: False`, with which the reference's forward returns no
`aux_outputs` (monodetr.py:270-283).  Pinned to the unmodified reference by tests/test_sizes_host.py (tests/golden/sizes.npz).

Training at other query counts: the reference's group self-attention hard-codes 50 queries per group
(depthaware_transformer.py:481-482: the rows before the last 11 x 50 are taken for denoising queries), so its training forward
fails at any num_queries but 50.  The oracle, like the product, splits the training queries into group_num groups of
num_queries each -- which is what the reference computes at 50 -- so the train-mode pins of those variants are the oracle's.

It also builds the criterion cases of tests/golden/criterion_sizes.npz: oracle/criterion.synthetic_case's head outputs and
targets with the number of valid targets of every image given exactly."""
import torch

from oracle import criterion as oc
from oracle import monodetr_torch as om
import oracle_dab as od          # tests/oracle_dab.py

# tag -> the model-section keys that differ from configs/monodetr.yaml
VARIANTS = {
    "deep": dict(enc_layers=6, dec_layers=6, dim_feedforward=1024),
    "q300": dict(num_queries=300, dim_feedforward=2048),
    "shallow": dict(enc_layers=1, dec_layers=1, aux_loss=False),
    "dab_q100": dict(use_dab=True, num_queries=100, dec_layers=4),
}


def sizes_cfg(tag):
    """The oracle's cfg of a variant: om.CFG with the variant's keys (use_dab / aux_loss included)."""
    return {**om.CFG, "use_dab": False, "aux_loss": True, **VARIANTS[tag]}


def deterministic_state_dict(cfg):
    return (od if cfg["use_dab"] else om).deterministic_state_dict(cfg)


def state_dict_spec(cfg):
    return od.state_dict_spec(cfg) if cfg["use_dab"] else om.state_dict_spec(cfg)


def forward(sd, images, calibs, img_sizes, training=False, cfg=None):
    """The reference's output dict at the cfg's sizes."""
    out = (od if cfg["use_dab"] else om).forward(sd, images, calibs, img_sizes, training=training, cfg=cfg)
    if not cfg["aux_loss"]:
        del out["aux_outputs"]
    return out


# name -> (seed, images' target counts, queries per group, group_num (1 = eval), decoder layers)
CRITERION_CASES = {
    "l6_q300_train": (31, (64, 0, 17), 300, 11, 6),      # 300 queries per group; an image with the most targets, one with none
    "l6_q100_eval": (32, (50, 1, 0), 100, 1, 6),
    "l6_q10_train": (33, (30, 0, 10), 10, 11, 6),        # more targets than queries: the rows are the queries
    "l1_q65_train": (34, (64, 63, 1), 65, 11, 1),        # one layer (aux_loss: False)
}
CRITERION_GMAX = 64


def criterion_case(name):
    """(head outputs with L - 1 aux outputs, padded targets) of a CRITERION_CASES entry."""
    seed, counts, nq, group, L = CRITERION_CASES[name]
    B = len(counts)
    out, padded = oc.synthetic_case(seed, B, nq * group, Gmax=CRITERION_GMAX, n_aux=L - 1, max_gt=1, empty_image=False)
    g = torch.Generator().manual_seed(seed + 1000)
    mask = torch.zeros(B, CRITERION_GMAX, dtype=torch.bool)
    for b, n in enumerate(counts):
        mask[b, torch.randperm(CRITERION_GMAX, generator=g)[:n]] = True      # valid rows are not a prefix
    padded["mask_2d"] = mask
    if L == 1:
        del out["aux_outputs"]
    return out, padded
