"""The voxel -> slot table of the masked voxel parameterisation (nsb_voxel_slots) and the kernels that index through it (nsb_masked_gather /
nsb_masked_scatter, nsb_compact_transpose, nsb_adam_masked_voxels), through the C entry points at synthetic sizes.

Every compact gradient and every fused Adam step lands in the voxel the table names, so a table that is wrong from some voxel on moves every later
parameter and no tolerance notices.  The table is three kernels: per-block counts (1024 voxels a block), a single-CTA exclusive scan of the counts in
chunks of 1024 blocks with a carry, and the write.  The sizes below sit on the warp, block and chunk seams (the carry only exists beyond
1024 * 1024 voxels); the reference is torch.cumsum on the CPU."""
import ctypes as C

import pytest
import torch

DEV = "cuda"
NSB_ERR_ARG = -1
BLOCK = 1024                       # voxels per count / write block, and block counts per chunk of the scan
CANARY = 0x1234ABCD                # a word no slot can be (the largest size here has 2.1 million voxels)

SIZES = [1, 31, 32, 33, 1023, 1024, 1025, BLOCK * BLOCK - 1, BLOCK * BLOCK, BLOCK * BLOCK + 1, 2 * BLOCK * BLOCK + 1025]
MASKS = ["ones", "zeros", "first", "last", "block_ends", "p01", "p50", "p99", "bytes_2_255"]


def make_mask(kind, n, seed=0):
    """uint8 [n] voxel mask of one of the kinds the table is checked with."""
    m = torch.zeros(n, dtype=torch.uint8)
    if kind == "ones":
        m.fill_(1)
    elif kind == "first":
        m[0] = 1
    elif kind == "last":
        m[n - 1] = 1
    elif kind == "block_ends":                      # one voxel per 1024-block, at the block's last position
        m[BLOCK - 1::BLOCK] = 1
    elif kind in ("p01", "p50", "p99"):
        p = {"p01": 0.01, "p50": 0.5, "p99": 0.99}[kind]
        m = (torch.rand(n, generator=torch.Generator().manual_seed(seed + n % 9973)) < p).to(torch.uint8)
    elif kind == "bytes_2_255":                     # any non-zero byte selects
        g = torch.Generator().manual_seed(seed + 1)
        m = torch.tensor([0, 2, 255, 1], dtype=torch.uint8)[torch.randint(0, 4, (n,), generator=g)]
    elif kind != "zeros":
        raise ValueError(kind)
    return m


def slot_reference(mask):
    """(slot_map int32 [n], count): slot_map[v] = how many selected voxels precede v, -1 where v is not selected."""
    sel = mask != 0
    incl = torch.cumsum(sel.to(torch.int64), 0)
    return torch.where(sel, incl - 1, torch.full_like(incl, -1)).to(torch.int32), int(incl[-1]) if mask.numel() else 0


# ------------------------------------------------------------------------------------ the reference itself (no GPU)
@pytest.mark.parametrize("n", [1, 33, 1025, 3 * BLOCK + 7])
@pytest.mark.parametrize("kind", MASKS)
def test_slot_reference_numbers_the_selected_voxels_in_order(kind, n):
    m = make_mask(kind, n)
    slots, count = slot_reference(m)
    idx = torch.nonzero(m).reshape(-1)                                   # an independent statement of the same thing
    assert count == idx.numel() and int((slots == -1).sum()) == n - count
    assert torch.equal(slots[idx], torch.arange(count, dtype=torch.int32))
    want = dict(ones=n, zeros=0, first=1, last=1, block_ends=n // BLOCK).get(kind)
    if want is not None:
        assert count == want
    if kind == "bytes_2_255" and n > 100:
        assert int((m == 2).sum()) > 0 and int((m == 255).sum()) > 0 and int((m == 0).sum()) > 0


# ------------------------------------------------------------------------------------ nsb_voxel_slots
def _lib():
    from nice_slam_b200 import _lib as lib
    return lib, lib.lib()


def run_voxel_slots(mask, tail=64):
    """-> (slot_map int32 [n] on the CPU, count, canary words behind slot_map)."""
    lib, L = _lib()
    n = mask.numel()
    m = mask.to(DEV)
    buf = torch.full((n + tail,), CANARY, dtype=torch.int32, device=DEV)
    cnt = torch.full((2,), CANARY, dtype=torch.int32, device=DEV)
    ws = torch.empty(L.nsb_voxel_slots_workspace(n), dtype=torch.uint8, device=DEV)
    lib.check(L.nsb_voxel_slots(m.data_ptr(), n, buf.data_ptr(), cnt.data_ptr(), ws.data_ptr(), ws.numel(), None), "nsb_voxel_slots")
    torch.cuda.synchronize()
    assert int(cnt[1]) == CANARY
    return buf[:n].cpu(), int(cnt[0]), buf[n:].cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", MASKS)
def test_voxel_slots_match_cumsum(kind, n):
    mask = make_mask(kind, n)
    want, want_count = slot_reference(mask)
    got, count, tail = run_voxel_slots(mask)
    assert count == want_count
    assert torch.equal(got == -1, mask == 0)
    if not torch.equal(got, want):
        bad = int(torch.nonzero(got != want)[0])
        pytest.fail("first wrong slot at voxel %d of %d (block %d): got %d, want %d" % (bad, n, bad // BLOCK, int(got[bad]), int(want[bad])))
    assert bool((tail == CANARY).all())


@pytest.mark.gpu
def test_voxel_slots_refuses_a_short_workspace_and_accepts_an_empty_grid():
    lib, L = _lib()
    n = 5 * BLOCK + 1
    need = L.nsb_voxel_slots_workspace(n)
    assert need >= 6 * 4
    m = torch.ones(n, dtype=torch.uint8, device=DEV)
    slots = torch.full((n,), CANARY, dtype=torch.int32, device=DEV)
    cnt = torch.full((1,), CANARY, dtype=torch.int32, device=DEV)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    assert L.nsb_voxel_slots(m.data_ptr(), n, slots.data_ptr(), cnt.data_ptr(), ws.data_ptr(), need - 1, None) == NSB_ERR_ARG
    assert L.nsb_voxel_slots(m.data_ptr(), -1, slots.data_ptr(), cnt.data_ptr(), ws.data_ptr(), need, None) == NSB_ERR_ARG
    torch.cuda.synchronize()
    assert int(cnt[0]) == CANARY and bool((slots == CANARY).all())        # a refusal launches nothing
    lib.check(L.nsb_voxel_slots(None, 0, None, cnt.data_ptr(), ws.data_ptr(), need, None), "nsb_voxel_slots(0)")
    torch.cuda.synchronize()
    assert int(cnt[0]) == 0


# ------------------------------------------------------------------------------------ gather / scatter / transpose / Adam through the table
GRID_SHAPES = [(5, 7, 11), (6, 3, 1)]               # D, H, W all different; and W = 1


def _grid(shape, layout, seed):
    D, H, W = shape
    val = torch.randn(1, 32, D, H, W, generator=torch.Generator().manual_seed(seed)).to(DEV)
    if layout == "channels_last":
        val = val.contiguous(memory_format=torch.channels_last_3d)
        if W == 1 or H == 1 or D == 1:              # size-1 dimensions leave the strides ambiguous: state them
            val = torch.empty_strided(val.shape, (32 * D * H * W, 1, 32 * H * W, 32 * W, 32), device=DEV).copy_(val)
        assert val.stride(1) == 1
    else:
        assert val.stride(4) == 1 and val.stride(1) == D * H * W
    return val


def _slots_of(vm):
    lib, L = _lib()
    n = vm.numel()
    m8 = vm.reshape(-1).to(DEV, torch.uint8)
    slots = torch.empty(n, dtype=torch.int32, device=DEV)
    cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
    ws = torch.empty(L.nsb_voxel_slots_workspace(n), dtype=torch.uint8, device=DEV)
    lib.check(L.nsb_voxel_slots(m8.data_ptr(), n, slots.data_ptr(), cnt.data_ptr(), ws.data_ptr(), ws.numel(), None), "nsb_voxel_slots")
    return slots, int(cnt)


def _transpose(src, n_sel, to_ref, tail=32):
    lib, L = _lib()
    dst = torch.full((32 * n_sel + tail,), float("nan"), device=DEV)
    lib.check(L.nsb_compact_transpose(src.data_ptr() if n_sel else None, dst.data_ptr() if n_sel else None, n_sel, int(to_ref), None), "nsb_compact_transpose")
    torch.cuda.synchronize()
    assert bool(torch.isnan(dst[32 * n_sel:]).all())                      # nothing behind dst is written
    return dst[:32 * n_sel]


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["channels_last", "ncdhw"])
@pytest.mark.parametrize("shape", GRID_SHAPES, ids=["5x7x11", "6x3x1"])
def test_masked_gather_scatter_on_a_non_cubic_grid(shape, layout):
    """compact = val[mask] and val[mask] = compact where a swapped pair of D, H, W would show (Mapper.py:324, :399, :517)."""
    from nice_slam_b200.renderer import grid_struct
    lib, L = _lib()
    val = _grid(shape, layout, 3)
    vm = torch.rand(shape, generator=torch.Generator().manual_seed(8)) < 0.3
    vm[0, 0, 0] = True; vm[-1, -1, -1] = True
    slots, count = _slots_of(vm)
    assert count == int(vm.sum())
    mask5 = vm.to(DEV)[None, None].repeat(1, 32, 1, 1, 1)                 # the reference's repeated mask, Mapper.py:319-320
    g = grid_struct(val)
    compact = torch.full((count + 1, 32), float("nan"), device=DEV)
    lib.check(L.nsb_masked_gather(C.byref(g), slots.data_ptr(), compact.data_ptr(), None), "nsb_masked_gather")
    assert torch.equal(compact[:count], val[0][:, vm.to(DEV)].t()) and bool(torch.isnan(compact[count]).all())
    assert torch.equal(_transpose(compact[:count].contiguous(), count, True), val[mask5])
    new = torch.randn(count, 32, generator=torch.Generator().manual_seed(2)).to(DEV)
    want = val.clone()
    want[mask5] = _transpose(new, count, True)
    before = val.clone()
    lib.check(L.nsb_masked_scatter(C.byref(g), slots.data_ptr(), new.data_ptr(), None), "nsb_masked_scatter")
    assert torch.equal(val, want) and torch.equal(val[~mask5], before[~mask5]) and not torch.equal(val, before)
    # nothing selected: both directions leave everything as it was
    none, zero = _slots_of(torch.zeros(shape, dtype=torch.bool))
    assert zero == 0 and bool((none == -1).all())
    keep, canary = val.clone(), torch.full((32,), float("nan"), device=DEV)
    lib.check(L.nsb_masked_scatter(C.byref(g), none.data_ptr(), canary.data_ptr(), None), "nsb_masked_scatter(0)")
    lib.check(L.nsb_masked_gather(C.byref(g), none.data_ptr(), canary.data_ptr(), None), "nsb_masked_gather(0)")
    assert torch.equal(val, keep) and bool(torch.isnan(canary).all())


@pytest.mark.gpu
@pytest.mark.parametrize("n_sel", [0, 1, 31, 32, 33, 1000])
def test_compact_transpose_both_ways(n_sel):
    """[n,32] slot-major <-> the reference's channel-major val[mask] order; 32 voxels per block, so 31 / 32 / 33 sit on the block seam."""
    src = torch.arange(32 * n_sel, dtype=torch.float32).view(n_sel, 32).to(DEV) + 0.5
    ref = _transpose(src, n_sel, True)
    assert torch.equal(ref.view(32, n_sel), src.t())
    back = _transpose(ref.contiguous(), n_sel, False)
    assert torch.equal(back.view(n_sel, 32), src)


@pytest.mark.gpu
def test_adam_step_through_the_slot_table_on_a_non_cubic_grid():
    """nsb_adam_masked_voxels over 5 x 7 x 11 with a sparse mask against torch.optim.Adam on val[mask] (Mapper.py:365-379), at the bar of the
    room-sized Adam test: a parameter stepped with another slot's gradient moves the wrong way by the learning rate, 1e4 times the bar."""
    from nice_slam_b200.renderer import grid_struct
    lib, L = _lib()
    shape = GRID_SHAPES[0]
    val = _grid(shape, "channels_last", 5)
    vm = torch.rand(shape, generator=torch.Generator().manual_seed(21)) < 0.15
    slots, count = _slots_of(vm)
    assert 10 < count < vm.numel() // 4
    mask5 = vm.to(DEV)[None, None].repeat(1, 32, 1, 1, 1)
    val_ref = val.clone()
    leaf = val_ref[mask5].clone().requires_grad_(True)
    opt = torch.optim.Adam([leaf], lr=0.01)
    em, ev = torch.zeros(count, 32, device=DEV), torch.zeros(count, 32, device=DEV)
    g = grid_struct(val)
    for step in (1, 2, 3):
        gv = torch.randn(count, 32, generator=torch.Generator().manual_seed(step)).to(DEV)
        leaf.grad = _transpose(gv, count, True).clone()
        opt.step()
        lib.check(L.nsb_adam_masked_voxels(C.byref(g), slots.data_ptr(), gv.data_ptr(), em.data_ptr(), ev.data_ptr(), 0.01, 0.9, 0.999, 1e-8, step, None),
                  "nsb_adam_masked_voxels")
        want = val_ref.clone()
        want[mask5] = leaf.detach()
        err = float((val - want).abs().max() / want.abs().max())
        assert err < 1e-6, (step, err)
        assert torch.equal(val[~mask5], val_ref[~mask5])
