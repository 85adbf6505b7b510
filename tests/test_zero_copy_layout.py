"""The zero-copy gradient buckets of hvd.DistributedOptimizer (shard_layout with one rank) for ResNet-50 and BERT-large
against golden layouts: bucket count, and per bucket its dtype, element count and every member's parameter and offset.
The fixture was recorded from the bucket packing that the zero-copy optimizer had before it shared shard_layout with
the sharded optimizer, so the layouts, which decide what each allreduce carries, must not move."""
import json
import os

import pytest
import torch

from horovod_b200 import models
from horovod_b200.torch.grad_buckets import shard_layout

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), 'golden', 'zero_copy_buckets.json')))


@pytest.mark.parametrize("cap_mb", [32, 1])
@pytest.mark.parametrize("model", ['resnet50', 'bert_large'])
def test_zero_copy_layout_matches_golden(model, cap_mb):
    with torch.device('meta'):
        params = list(getattr(models, model)().parameters())
    buckets = shard_layout([[(p.numel(), p.dtype) for p in params]], 1, cap_mb * 1024 * 1024)
    got = [{'dtype': str(b['dtype']).replace('torch.', ''), 'numel': b['numel'],
            'members': [[i, off] for i, off, numel in b['members']]} for b in buckets]
    want = GOLDEN[model][str(cap_mb)]
    assert len(got) == len(want)
    assert got == want
