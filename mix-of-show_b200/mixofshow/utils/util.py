"""Drop-in for the parts of the reference's `mixofshow/utils/util.py` that `test_edlora.py` and the validation pass of
`train_edlora.py` use: `NEGATIVE_PROMPT`, `pil_imwrite`, `draw_prompt` and `compose_visualize`."""
import os
import os.path as osp

import numpy as np
from PIL import Image, ImageDraw, ImageFont

NEGATIVE_PROMPT = 'longbody, lowres, bad anatomy, bad hands, missing fingers, extra digit, fewer digits, cropped, worst quality, low quality'

GRID_PADDING = 2            # torchvision make_grid's default padding (zero-valued)


def pil_imwrite(img, file_path, auto_mkdir=True):
    """Saves a PIL image, creating the parent directory when `auto_mkdir`."""
    assert isinstance(img, Image.Image), 'model should return a list of PIL images'
    if auto_mkdir:
        os.makedirs(osp.abspath(osp.dirname(file_path)), exist_ok=True)
    img.save(file_path)


def draw_prompt(text, height, width, font_size=45):
    """A white `width` x `height` tile with `text` in black, wrapped every `guess_count` characters, where
    `guess_count` is the longest prefix that fits in 80% of the width.

    The layout is the reference's; the font is Pillow's scalable default font instead of the reference's bundled
    arial.ttf, so these tiles differ from the reference's by the glyphs only."""
    img = Image.new('RGB', (width, height), (255, 255, 255))
    draw = ImageDraw.Draw(img)
    font = ImageFont.load_default(size=font_size)
    guess_count = 0
    while font.getlength(text[:guess_count]) + 0.1 * width < width - 0.1 * width and guess_count < len(text):
        guess_count += 1
    text_new = ''
    for idx, s in enumerate(text):
        if idx % guess_count == 0:
            text_new += '\n'
            if s == ' ':
                s = ''              # a new line drops its leading space
        text_new += s
    draw.text([int(0.1 * width), int(0.3 * height)], text_new, font=font, fill='black')
    return img


def make_grid(tiles, nrow, padding=GRID_PADDING):
    """torchvision `make_grid` geometry for equally sized [H, W, C] uint8 tiles: `nrow` tiles per row, `padding` zero
    pixels around and between them."""
    h, w, c = tiles[0].shape
    xmaps = min(nrow, len(tiles))
    ymaps = -(-len(tiles) // xmaps)
    ph, pw = h + padding, w + padding
    grid = np.zeros((ph * ymaps + padding, pw * xmaps + padding, c), dtype=np.uint8)
    for k, t in enumerate(tiles):
        y, x = divmod(k, xmaps)
        grid[y * ph + padding:y * ph + padding + h, x * pw + padding:x * pw + padding + w] = t
    return grid


def compose_grid(dir_path):
    """The grid `compose_visualize` writes and its file name.  Files are `{prompt}---{sample_args}---{index}---{suffix}`
    in `sorted(os.listdir)` order; each new prompt is preceded by a `draw_prompt` tile."""
    img_list = []
    prompts, sample_args, suffixes = set(), set(), set()
    for filename in sorted(os.listdir(dir_path)):
        prompt, args, _, suffix = osp.splitext(osp.basename(filename))[0].split('---')
        img = np.asarray(Image.open(osp.join(dir_path, filename)))
        height, width = img.shape[:2]
        if prompt not in prompts:
            img_list.append(np.asarray(draw_prompt(prompt, height=height, width=width, font_size=45)))
        prompts.add(prompt)
        sample_args.add(args)
        suffixes.add(suffix)
        img_list.append(img)
    assert len(sample_args) == 1, 'compose dir should contain images form same sample args.'
    assert len(suffixes) == 1, 'compose dir should contain images form same suffix.'
    grid = make_grid(img_list, nrow=len(img_list) // len(prompts))
    return grid, f'{sample_args.pop()}---{suffixes.pop()}.jpg'


def compose_visualize(dir_path):
    """Writes one JPEG grid of the images in `dir_path` (a row per prompt: the prompt's text tile, then its samples)
    next to the directory, as `{sample_args}---{suffix}.jpg`."""
    grid, save_name = compose_grid(dir_path)
    Image.fromarray(grid).save(osp.join(osp.dirname(dir_path), save_name))
