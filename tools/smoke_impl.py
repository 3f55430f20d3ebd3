"""smoke(): ONE small invocation of the hot path on cuda:0, checked against the CPU oracle.

Order matters for the driver's launch trace (it records the first ~1000 kernel launches): the hand-written kernels run
FIRST, called directly through the C ABI (INT8 wgmma GEMM, implicit-GEMM conv3x3, GEGLU epilogue, small-Tk / mma.sync
attention, GroupNorm, LayerNorm, quantizer) and checked against the op oracle; only then the SD-style tiny UNet
fixture (spatial transformer + cross attention, asymmetric W4A8, sm_abit 16, split shortcut) is folded (torch ops on
the GPU: load-time only) and run through QuantModel.forward and two PLMS steps of the sampler."""
import torch


def run():
    from tests import test_ops_gpu as T
    from tests.test_oracle_golden import load_case, noise_band_mse, oracle_forward
    from tests.test_unet_gpu import build_qnn
    from qdiff_b200 import _lib, samplers
    dev = torch.device("cuda:0")
    L = _lib.lib()
    n0 = L.qd_launch_count()
    # ---- direct kernel calls through the C ABI, each checked against the op oracle (same functions as the GPU tests)
    T.test_qgemm_plain(dev, 300, 320, 320, True)
    T.test_qconv3x3(dev, 2, 16, 16, 64, 96, True)
    T.test_qgemm_geglu_fused(dev)
    for args in ((2, 8, 40, 256, 256, False, 16), (2, 8, 40, 200, 77, False, 16), (1, 2, 160, 64, 64, False, 16)):
        T.test_qattention(dev, *args)
    n_direct = L.qd_launch_count() - n0
    assert n_direct >= 6, "direct kernel calls did not go through libqdiff_b200.so"
    # ---- the UNet path
    g = load_case("sd_tiny_w4a8_sm16")
    qnn = build_qnn(g, dev)
    n0 = L.qd_launch_count()
    out = qnn(g["x"].to(dev), g["t"].to(dev), g["context"].to(dev)).cpu()
    n1 = L.qd_launch_count()
    ref = oracle_forward(g)
    mse = ((out.double() - ref.double()) ** 2).mean().item()
    band = noise_band_mse(g, ref)
    assert torch.isfinite(out).all()
    assert n1 > n0, "no kernels were launched through libqdiff_b200.so"
    assert mse <= max(2 * band, 1e-6), f"smoke parity failed: mse {mse:.3e} vs noise band {band:.3e}"
    sampler = samplers.PLMSSampler(qnn, samplers.Schedule("linear", 1000, 0.00085, 0.0120))
    x, _ = sampler.sample(S=2, batch_size=2, shape=(4, 16, 16), conditioning=g["context"].to(dev),
                          unconditional_guidance_scale=1.0, x_T=g["x"])
    assert torch.isfinite(x).all()
    print(f"smoke ok: {n_direct} direct kernel launches checked against the op oracle; UNet eps mse vs oracle {mse:.3e} "
          f"(reference fp32 noise band {band:.3e}); {n1 - n0} kernels launched via the C ABI; 2-step PLMS latent finite")


if __name__ == "__main__":
    run()
