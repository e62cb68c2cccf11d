"""GPU numerics of individual embedding / elementwise kernels vs the PyTorch fp32 reference paths."""
import pytest
import torch

from hugectr_b200.embedding import ops as E

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("act", [torch.bfloat16, torch.float32])
def test_dp_dense_wgrad_privatized_and_global(act):
    """data-parallel dense wgrad (csrc/embedding.cu emb_dp_wgrad_kernel): tiny tables take the
    shared-memory privatised path, larger ones the global-reduction path"""
    torch.manual_seed(3)
    b, ev = 777, 64
    rows = [5, 300, 9000, 40]
    hot = [1, 3, 4, 2]
    comb = [0, 1, 0, 1]
    lookups, koff, goff, roff = [], 0, 0, 0
    for r, h, c in zip(rows, hot, comb):
        lookups.append(E.LookupDesc(table_row_off=roff, key_off=koff, out_off=goff, grad_off=goff,
                                    hotness=h, key_stride=h, num_shards=1, shard_idx=0, out_stride=ev,
                                    grad_stride=ev, combiner=c, ev_size=ev, rows=r))
        koff += b * h
        goff += b * ev
        roff += r
    keys = torch.cat([torch.randint(0, r, (b * h,), dtype=torch.int32) for r, h in zip(rows, hot)])
    # skew: most samples of the first tables hit row 0 (hot-row contention)
    keys[:b // 2] = 0
    grad = torch.randn(goff).to(act)
    table = torch.zeros(roff * ev)
    ref = torch.zeros(roff * ev)
    E.backward_accum(lookups, None, table, ev, [keys], [grad.float()], b, None, 0.5, dense_wgrad=ref)
    dev = torch.device("cuda")
    out = torch.zeros(roff * ev, device=dev)
    ld = E.lookups_to_device(lookups, dev)
    E.backward_accum(lookups, ld, table.to(dev), ev, [keys.to(dev)], [grad.to(dev)], b, None, 0.5,
                     dense_wgrad=out, key_bytes=4, act_bf16=(act == torch.bfloat16))
    torch.cuda.synchronize()
    err = (out.cpu() - ref).abs().max().item()
    assert err < 2e-3 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize("ev,shards", [(128, 8), (64, 3), (16, 2), (256, 4)])
def test_forward_row_sharded_compacted_gather(ev, shards):
    """row-sharded lookups take the compacted-gather path of emb_fwd_kernel (ballot over up to 4 keys
    per lane); compare one shard's partial pooling with the PyTorch reference"""
    torch.manual_seed(5)
    b = 333
    specs = [(5000, 100, 0), (900, 7, 1), (77, 1, 0), (4000, 27, 1)]   # (vocab, hotness, combiner)
    shard = shards - 1
    lookups, koff, ooff, roff = [], 0, 0, 0
    for vocab, h, c in specs:
        rows = (vocab - shard + shards - 1) // shards
        lookups.append(E.LookupDesc(table_row_off=roff, key_off=koff, out_off=ooff, grad_off=ooff,
                                    hotness=h, key_stride=h, num_shards=shards, shard_idx=shard,
                                    out_stride=ev, grad_stride=ev, combiner=c, ev_size=ev, rows=rows))
        koff += b * h
        ooff += b * ev
        roff += rows
    # one unsharded lookup in the same launch (regular path)
    lookups.append(E.LookupDesc(table_row_off=roff, key_off=koff, out_off=ooff, grad_off=ooff, hotness=5,
                                key_stride=5, num_shards=1, shard_idx=0, out_stride=ev, grad_stride=ev,
                                combiner=0, ev_size=ev, rows=600))
    keys = torch.cat([torch.randint(0, v, (b * h,), dtype=torch.int32) for v, h, _ in specs] +
                     [torch.randint(0, 600, (b * 5,), dtype=torch.int32)])
    ooff += b * ev
    roff += 600
    table = torch.randn(roff * ev)
    ref = torch.zeros(ooff)
    E.forward(lookups, None, table, ev, [keys], [ref], b)
    dev = torch.device("cuda")
    out = torch.zeros(ooff, device=dev)
    E.forward(lookups, E.lookups_to_device(lookups, dev), table.to(dev), ev, [keys.to(dev)], [out], b,
              key_bytes=4, act_bf16=False)
    torch.cuda.synchronize()
    err = (out.cpu() - ref).abs().max().item()
    assert err < 1e-3 * max(1.0, ref.abs().max().item()), err
