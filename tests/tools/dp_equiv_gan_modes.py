"""tests/tools/dp_equiv.py with the `--gan_mode` of both models taken from SN_DP_GAN_MODE (default vanilla): 2-rank
CUDA data-parallel gradients and losses against the single-process full batch, under torchrun, for each objective.
Every GAN term is a per-call batch mean, so equal shards plus gradient averaging reproduce the full-batch step."""
import os

import dp_equiv

MODE = os.environ.get("SN_DP_GAN_MODE", "vanilla")
_opt = dp_equiv._opt
dp_equiv._opt = lambda B, S, **over: _opt(B, S, **{"gan_mode": MODE, **over})

if __name__ == "__main__":
    print(f"gan_mode={MODE}", flush=True)
    dp_equiv.main()
