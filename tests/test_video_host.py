"""GIF palettes and picture files without a GPU: known answers of the quantiser's numpy restatement (oracle/palette_oracle.py), the Pillow
round trip of indexed frames, the header's section 11 and the refusal of CPU tensors."""
import numpy as np
import pytest
import torch


def test_oracle_single_colour_gives_one_entry():
    from oracle import palette_oracle as po
    frames = np.broadcast_to(np.array([10, 200, 37], np.uint8), (2, 9, 11, 3)).copy()
    pal, nc, idx = po.quantize(frames, 256)
    assert nc.tolist() == [1, 1] and (idx == 0).all()
    assert pal[0, 0].tolist() == [10, 200, 37] and not pal[:, 1:].any()


def test_oracle_reproduces_few_colours_in_distinct_cells():
    from oracle import palette_oracle as po
    rng = np.random.default_rng(0)
    colours = np.array([[0, 0, 0], [255, 255, 255], [255, 0, 0], [8, 16, 24], [100, 150, 200], [37, 250, 3], [64, 64, 64]], np.uint8)
    assert len({tuple(c >> 3) for c in colours}) == len(colours)
    frame = colours[rng.integers(0, len(colours), (23, 31))]
    for colors in (len(colours), 256):
        pal, nc, idx = po.quantize(frame[None], colors)
        assert nc[0] == len(colours)
        assert np.array_equal(pal[0][idx[0]], frame)
        assert sorted(map(tuple, pal[0, :nc[0]].tolist())) == sorted(map(tuple, colours.tolist()))


def test_oracle_mean_rounds_half_up():
    from oracle import palette_oracle as po
    frame = np.zeros((1, 2, 2, 3), np.uint8)
    frame[0, :, 0] = 8                                  # one cell (1, 1, 1) holding 8 twice and 9 twice: mean 8.5 -> 9
    frame[0, :, 1] = 9
    pal, nc, idx = po.quantize(frame, 256)
    assert nc[0] == 1 and pal[0, 0].tolist() == [9, 9, 9]


def test_oracle_tie_maps_to_lower_index():
    from oracle import palette_oracle as po
    palette = np.zeros((256, 3), np.uint8)
    palette[0], palette[1] = [10, 10, 10], [20, 20, 20]
    frame = np.array([[[15, 15, 15], [16, 16, 16], [14, 14, 14]]], np.uint8)
    assert po.nearest(frame, palette, 2).tolist() == [[0, 1, 0]]
    palette[0], palette[1] = [20, 20, 20], [10, 10, 10]
    assert po.nearest(frame, palette, 2).tolist() == [[0, 0, 1]]


def test_oracle_two_clusters_with_two_colours():
    from oracle import palette_oracle as po
    rng = np.random.default_rng(1)
    frame = np.where(rng.random((32, 32, 1)) < 0.5, rng.integers(0, 40, (32, 32, 3)), rng.integers(200, 256, (32, 32, 3))).astype(np.uint8)
    pal, nc, idx = po.quantize(frame[None], 2)
    assert nc[0] == 2
    bright = frame.astype(int).sum(-1) > 300
    assert (idx[0][bright] == idx[0][bright][0]).all() and (idx[0][~bright] == idx[0][~bright][0]).all()
    assert idx[0][bright][0] != idx[0][~bright][0]
    # every box is split at its median: the upper half of the split is appended, the lower keeps index 0
    assert pal[0, 0].max() < 40 and pal[0, 1].min() >= 200


def test_oracle_stops_when_nothing_is_splittable():
    from oracle import palette_oracle as po
    frame = np.zeros((1, 4, 4, 3), np.uint8)
    frame[0, :2] = [1, 2, 3]                            # two colours in one cell: one unsplittable box
    frame[0, 2:] = [250, 3, 3]
    pal, nc, _ = po.quantize(frame, 256)
    assert nc[0] == 2 and pal[0, 0].tolist() == [1, 2, 3] and pal[0, 1].tolist() == [250, 3, 3]


def test_pillow_round_trip_of_indexed_frames(tmp_path):
    """what write_gif does with the quantiser's output: distinct P frames with their own palettes decode frame by frame to palette[indices]"""
    from PIL import Image
    from oracle import palette_oracle as po
    rng = np.random.default_rng(2)
    frames = np.zeros((5, 24, 40, 3), np.uint8)
    for b in range(5):
        frames[b, 4 + b:16 + b, 6:30] = rng.integers(0, 256, (12, 24, 3))
    pal, nc, idx = po.quantize(frames, 256)
    images = []
    for b in range(5):
        im = Image.frombytes('P', (40, 24), idx[b].tobytes())
        im.putpalette(pal[b, :nc[b]].tobytes())
        images.append(im)
    path = tmp_path / 'x.gif'
    images[0].save(path, save_all=True, append_images=images[1:], duration=200, loop=0)
    with Image.open(path) as im:
        assert im.n_frames == 5 and im.info['loop'] == 0
        for b in range(5):
            im.seek(b)
            assert im.info['duration'] == 200
            assert np.array_equal(np.asarray(im.convert('RGB')), pal[b][idx[b]]), b


def test_header_declares_the_palette_entry_points():
    from sparsefusion_b200 import _lib
    protos = _lib.parse_header()
    assert protos['sfb_palette_work_bytes'] == ('uint64_t', ['int B', 'int H', 'int W'])
    ret, args = protos['sfb_palette_quantize']
    assert ret == 'int' and len(args) == 10 and args[0] == 'const uint8_t* rgb' and args[-1] == 'void* stream'


def test_video_refuses_cpu_tensors(tmp_path):
    from sparsefusion_b200 import video
    x = torch.zeros(2, 8, 8, 3, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match='CUDA'):
        video.quantize_palette(x)
    with pytest.raises(RuntimeError, match='CUDA'):
        video.write_gif(str(tmp_path / 'a.gif'), x)
    with pytest.raises(RuntimeError, match='CUDA'):
        video.write_jpeg(str(tmp_path / 'a.jpg'), x[0])
    with pytest.raises(RuntimeError, match='CUDA'):
        video.to_uint8(torch.zeros(2, 8, 8, 3))
    assert not list(tmp_path.iterdir())
