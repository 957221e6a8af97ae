"""2-rank equivalence of `--b200_sync_bn 1` for the two models on a bare U-Net (run under torchrun;
tests/test_unet_gpu.py launches it): pix2pix with --norm batch, and the texture stage with --netG unet_128 and
--norm instance, where only the generator has batch norm.  The checks and the printed lines are those of
sync_bn_equiv.py, whose driver this reuses with these two configurations."""
import gc
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import sync_bn_equiv as SE  # noqa: E402
import torch.distributed as dist  # noqa: E402


def stage_opt(stage, B, S, **over):
    if stage == "pix2pix":
        return SE._opt(B, S, model="pix2pix", netG="unet_128", norm="batch", lambda_l1=10.0, beta1=0.5, lr=2e-4,
                       **over)
    return SE._opt(B, S, model="texture", netG="unet_128", norm="instance", lambda_l1=10, lambda_content=0,
                   lambda_style=0, **over)


def batch_of(stage, B, S):
    if stage == "pix2pix":
        _, _, cloth, tgt = SE.synth_texture_batch(B, S)
        return dict(cloths=cloth, target_textures=tgt)
    return SE.batch_of("texture", B, S)


def main():
    texture_batch = SE.batch_of
    SE.stage_opt = stage_opt
    SE.batch_of = lambda stage, B, S: batch_of(stage, B, S) if stage == "pix2pix" else texture_batch("texture", B, S)
    ok = SE.run("pix2pix", 128, 2)
    gc.collect()
    ok &= SE.run("texture_unet_128", 128, 2)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
