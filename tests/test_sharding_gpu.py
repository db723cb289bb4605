"""SURVEY 4 item 4 / 8e on hardware: with images sharded over 2 GPUs (NCCL, weights broadcast once from rank 0, nothing
exchanged per step) every image's final latents are BIT-IDENTICAL to the same image run alone on one GPU.  Needs two
GPUs; skipped on a one-GPU machine."""
import math
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _images(dev):
    from paint_with_words_sd_b200 import conditioning as C
    from paint_with_words_sd_b200.scheduler import LMSDiscreteScheduler
    from paint_with_words_sd_b200.synthetic import RandomTextEncoder, SimpleWordTokenizer
    from paint_with_words_sd_b200.unet import UNetConfig
    from tests.fixtures import SETTINGS, color_map_image
    cfg = UNetConfig.tiny()
    tok, enc = SimpleWordTokenizer(), RandomTextEncoder(cfg.cross_attention_dim).to(dev)
    sch = LMSDiscreteScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
    sch.set_timesteps(3)
    out = []
    for i, name in enumerate(("aurora", "cat_dog")):
        s = SETTINGS[name]
        _, _, c, u = C._encode_text_color_inputs(enc, tok, dev, color_map_image(name, 128), dict(s["ctx"]), s["prompt"], "")
        lat = torch.randn(1, 4, 16, 16, generator=torch.manual_seed(i)) * sch.init_noise_sigma
        out.append((c, u, lat))
    return cfg, sch, out


WF = lambda w, sigma, qk: 0.4 * w * math.log(1 + sigma) * qk.max()   # noqa: E731


def _worker(rank, world, port, ret):
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import paint_with_words_sd_b200 as P
    from paint_with_words_sd_b200 import sharding
    from paint_with_words_sd_b200.pipeline import PwWSampler
    from paint_with_words_sd_b200.unet import build_unet
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    assert sharding.init_distributed("nccl")
    cfg, sch, imgs = _images(dev)
    unet = build_unet(cfg, seed=0 if rank == 0 else 123, dtype=torch.float16, device=dev)   # replicas differ until the broadcast
    nbytes = sharding.broadcast_module_weights(unet, src=0)
    P.patch_unet(unet)
    try:
        mine = sharding.shard_images(len(imgs), rank, world)
        local = {}
        for i in mine:
            c, u, lat = imgs[i]
            local[i] = PwWSampler(unet, sch, [c], [u], lat.to(dev), WF, 7.5, use_graph=False).run().clone()
        allv = sharding.gather_latents(local, len(imgs))
        if rank == 0:                                   # the same images, alone, on this one GPU
            solo = [PwWSampler(unet, sch, [c], [u], lat.to(dev), WF, 7.5, use_graph=False).run().clone() for (c, u, lat) in imgs]
            ret["equal"] = [bool(torch.equal(allv[i].to(dev), solo[i])) for i in range(len(imgs))]
            ret["nbytes"] = nbytes
    finally:
        P.unpatch_all()
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpu_sharding_is_bit_identical_per_image():
    world, port = 2, _free_port()
    with mp.Manager() as mgr:
        ret = mgr.dict()
        mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
        equal, nbytes = list(ret["equal"]), int(ret["nbytes"])
    assert nbytes > 0 and all(equal), equal
