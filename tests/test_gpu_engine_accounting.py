"""What the engine reports about its own work: plip_launch_count (bench.py's gpu_launches), the per-role profile rows
(bench.py's roofline / kernels_in_step), and the shared scratch of the handle-free similarity entry points."""
import threading

import pytest
import torch

from oracle import synth
from plip_b200._lib import lib
from plip_b200.engine import similarity_topk

pytestmark = pytest.mark.gpu

VIS = dict(S=50, D=768, FF=3072)
TXT = dict(S=77, D=512, FF=2048)
MICRO_BATCHES_150 = (64, 64, 22)        # n = 150 on the max_micro_batch = 64 engine: three eager passes


@pytest.fixture(scope="module")
def images():
    return torch.from_numpy(synth.tiles_u8(150, seed=71)).cuda()


@pytest.fixture(scope="module")
def captions():
    ids, mask = synth.token_ids(150, seed=72)
    return ids.cuda(), mask.cuda()


@pytest.fixture
def pruning(engine, request):
    engine.set_last_layer_pruning(request.param)
    yield request.param
    engine.set_last_layer_pruning(False)


def _launches(call):
    before = lib().plip_launch_count()
    call()
    return lib().plip_launch_count() - before


@pytest.mark.parametrize("pruning", [False, True], indirect=True)
@pytest.mark.parametrize("normalize", [False, True])
def test_image_launch_count(engine, images, normalize, pruning):
    """im2col, patch GEMM, class rows, pre-LN, row statistics, 12 x 5, pooled LN, projection = 67 kernels per
    micro-batch, + l2 normalisation, + the pooled-row gather of a pruned last layer.  Graph capture, graph replay
    (n = 8) and eager micro-batches (n = 150) count the same kernels."""
    per_pass = 67 + normalize + pruning
    for _ in range(2):                  # a new graph key: eager run + capture, then a replay
        assert _launches(lambda: engine.encode_images(images[:8], normalize=normalize)) == per_pass
    assert _launches(lambda: engine.encode_images(images, normalize=normalize)) == 3 * per_pass


@pytest.mark.parametrize("pruning", [False, True], indirect=True)
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("masked", [False, True])
def test_text_launch_count(engine, captions, masked, normalize, pruning):
    """Token embedding + eos search (2), row statistics, 12 x 5, pooled LN, projection = 65 kernels per micro-batch,
    + mask conversion, + l2 normalisation, + the pooled-row gather of a pruned last layer."""
    ids, mask = captions
    per_pass = 65 + masked + normalize + pruning
    for _ in range(2):
        assert _launches(lambda: engine.encode_text(ids[:8], mask[:8] if masked else None, normalize=normalize)) == per_pass
    assert _launches(lambda: engine.encode_text(ids, mask if masked else None, normalize=normalize)) == 3 * per_pass


def _gemm_work(M, N, K, out_bytes, xb_out):
    """2·M·N·K FLOPs; A and W read once, the output written once (fp32 residual: read + write), + the 16-bit copy."""
    return 2 * M * N * K, M * K * 2 + N * K * 2 + M * N * out_bytes + (M * N * 2 if xb_out else 0)


def _expected_rows(tower, pruned):
    """{row name: (launches, gemm flops, gemm bytes)} of one un-normalised call at n = 150 (flops / bytes: GEMMs only)."""
    d = VIS if tower == "vision" else TXT
    S, D, FF = d["S"], d["D"], d["FF"]
    rows = {}

    def add(role, launches=1, work=(0, 0)):
        n0, f0, b0 = rows.get(role, (0, 0, 0))
        rows[role] = (n0 + launches, f0 + work[0], b0 + work[1])

    for mb in MICRO_BATCHES_150:
        M = mb * S
        if tower == "vision":
            add("im2col")
            add("gemm[patch_embed]", work=_gemm_work(mb * 49, D, 3072, 4, False))
            add("misc")                                                   # class rows
            add("layernorm")                                              # pre-LN
        else:
            add("text_embed")
        add("rowstats_cast")
        for layer in range(12):
            last = layer == 11
            add("gemm[ln1+qkv]", work=_gemm_work(M, 3 * D, D, 2, False))
            add("attention")
            rows_tail = mb if (pruned and last) else M
            if pruned and last:
                add("misc")                                               # pooled-row gather
            add("gemm[out_proj+resid]", work=_gemm_work(rows_tail, D, D, 8, True))
            add("gemm[ln2+fc1+gelu]", work=_gemm_work(rows_tail, FF, D, 2, False))
            add("gemm[fc2+resid]", work=_gemm_work(rows_tail, D, FF, 8, not last))
        add("layernorm")                                                  # pooled rows
        add("gemm[projection]", work=_gemm_work(mb, 512, D, 4, False))
    return {f"{tower}/{k}": v for k, v in rows.items()}


@pytest.mark.parametrize("pruning", [False, True], indirect=True)
def test_profile_rows_follow_the_layer_structure(engine, images, captions, pruning):
    engine.profile(True)
    try:
        engine.encode_images(images)
        engine.encode_text(captions[0])
        got = {r["name"]: r for r in engine.profile_read()}
    finally:
        engine.profile(False)
    want = {**_expected_rows("vision", pruning), **_expected_rows("text", pruning)}
    assert sorted(got) == sorted(want)
    for name, (launches, flops, nbytes) in want.items():
        assert got[name]["launches"] == launches, name
        if name.split("/")[1].startswith("gemm["):
            assert got[name]["flops"] == pytest.approx(flops, rel=1e-12), name
            assert got[name]["bytes"] == pytest.approx(nbytes, rel=1e-12), name


def test_similarity_topk_from_two_threads_on_two_streams():
    """Tensor-core top-k (n >= 256, m >= 8192): two host threads on two streams share the per-device scratch pools
    and must each get the serial result."""
    g = torch.Generator().manual_seed(73)
    space = torch.randn(20000, 512, generator=g).cuda()
    queries = [torch.randn(n, 512, generator=g).cuda() for n in (300, 700)]
    serial = [similarity_topk(q, space, 20) for q in queries]
    torch.cuda.synchronize()
    results = [None, None]
    start = threading.Barrier(2)

    def work(i):
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            start.wait()
            results[i] = similarity_topk(queries[i], space, 20)
            stream.synchronize()

    threads = [threading.Thread(target=work, args=(i,)) for i in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for (idx, val), (ref_idx, ref_val) in zip(results, serial):
        assert torch.equal(idx, ref_idx) and torch.equal(val, ref_val)
