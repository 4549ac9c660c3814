"""Host-side dispatch heuristics of the tensor-core GEMM (pure Python, no GPU): pinned to the shapes they were
tuned on so a refactor cannot silently change a measured path."""
import torch

from baton_b200.ops import functional as F
from baton_b200.ops import nn as bnn


def test_tile_width_tracks_the_wave_count():
    assert F.pick_bn(8192, 8192) == 128          # big GEMM: the widest tile the kernels instantiate
    assert F.pick_bn(16384, 2304) == 128         # BERT qkv at batch 128 x seq 128
    assert F.pick_bn(4096, 768) == 128           # 32 x 6 = 192 tiles of 128
    assert F.pick_bn(8192, 64) == 64             # ResNet layer1
    assert F.pick_bn(128, 512) == 64             # ResNet layer4 at 32x32 inputs: few rows, keep CTAs many


def test_cluster_split_k_only_for_deep_few_tile_problems():
    # (M, N, K) of the ResNet-18 forward GEMMs at batch 128, 32x32 inputs
    assert F.pick_cluster_k(8192, 64, 576, 64) == 1          # layer1: 9 k-tiles, plenty of tiles
    assert F.pick_cluster_k(2048, 128, 1152, 64) == 4        # layer2
    assert F.pick_cluster_k(512, 256, 2304, 64) == 4         # layer3
    assert F.pick_cluster_k(128, 512, 4608, 64) == 8         # layer4: 8 tiles x 8 = 64 CTAs <= half the SMs
    assert F.pick_cluster_k(8192, 8192, 8192, 128) == 1      # never for problems that fill the machine


def test_atomic_split_k_for_weight_gradients():
    # wgrad dW[Cout, K] over M = N*Ho*Wo pixels: few tiles, very long reduction
    assert F.pick_split_k(64, 576, 8192, 64) > 1
    assert F.pick_split_k(3072, 768, 16384, 128) == 1        # BERT ffn wgrad already has 144 tiles
    assert F.pick_split_k(128, 128, 256, 64) == 1            # short K: nothing to split


def test_fused_statistics_need_a_tma_legal_k():
    assert F.gemm_stats_fusable(8192, 64, 576)
    assert F.gemm_stats_fusable(2048, 128, 1152)             # cluster split-K reduces the statistics in DSMEM
    assert not F.gemm_stats_fusable(32768, 64, 147)          # un-padded stem K would go to the SIMT kernel


def test_conv_only_offers_statistics_workspace_when_training_with_a_linked_batchnorm():
    conv = bnn.Conv2d(64, 64, 3, 1, 1)
    x = torch.zeros(4, 8, 8, 64)
    assert conv._fusable_stats(x) is None                    # no BatchNorm linked
    ws = torch.zeros(4 * 64)
    conv.bn_ws = ws
    got = conv._fusable_stats(x)
    assert got is not None and got.data_ptr() == ws.data_ptr() and got.numel() == 2 * 64
    conv.eval()
    assert conv._fusable_stats(x) is None                    # running statistics in eval mode
    conv.train()
    with torch.no_grad():
        assert conv._fusable_stats(x) is None                # inference pass
