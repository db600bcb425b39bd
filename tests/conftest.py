import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def tiny_cfg():
    return dict(use_bfloat16=True, hidden_size=128, vocab_size=1000, patch_size=16, spatial_pool_size=2, num_attention_heads=2,
                num_hidden_layers=2, num_vision_transformer_hidden_layers=2, num_lang_transformer_hidden_layers=2,
                intermediate_size=256, initializer_range=0.02, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.0,
                max_position_embeddings=64, num_chunks_in_group=2, do_projection=True, do_bias=True, contrastive_size=128,
                contrast_coef=0.25, contrast_temp=0.05, image_shuffle_prob=0.4, masking_rate=0.2, resnet_layers=[])
