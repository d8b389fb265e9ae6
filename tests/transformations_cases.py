"""The transformations of tests/golden/make_transformations_golden.py, built from either class set: ``m`` holds the modules
``geo`` (object_detection_2d_geometric_ops), ``patch`` (_patch_sampling_ops), ``photo`` (_photometric_ops) and ``valid``
(_image_boxes_validation_utils), the reference's or this package's, so that both sides construct the same objects.

``SINGLES``: every class of the op modules that had no planner before, each alone behind ``ConvertTo3Channels`` (and the dtype
or colour conversions the reference's class expects).  ``CHAINS``: custom chains through ``DataGenerator.generate``, each with
its dataset (tests/chain_dataset.py), labels dtype, seed and number of batches of ``BATCH``."""
import chain_dataset as ds

BATCH = 4


def _bf(m):
    return m.valid.BoxFilter(check_overlap=True, check_min_area=True, check_degenerate=True, overlap_criterion='center_point',
                             overlap_bounds=(0.3, 1.0), min_area=9)


def _iv(m):
    return m.valid.ImageValidator(overlap_criterion='area', bounds=(0.5, 1.0), n_boxes_min=1)


def _f32(m):
    return m.photo.ConvertDataType('float32')


def _u8(m):
    return m.photo.ConvertDataType('uint8')


def _hsv(m):
    return m.photo.ConvertColor('RGB', 'HSV')


def _rgb(m):
    return m.photo.ConvertColor('HSV', 'RGB')


SINGLES = {
    'flip_h': lambda m: [m.geo.Flip('horizontal')],
    'flip_v': lambda m: [m.geo.Flip('vertical')],
    'translate': lambda m: [m.geo.Translate(0.2, -0.1, clip_boxes=True, box_filter=_bf(m), background=(10, 20, 30))],
    'translate_noclip': lambda m: [m.geo.Translate(-0.25, 0.3, clip_boxes=False)],
    'scale_in': lambda m: [m.geo.Scale(1.3, box_filter=_bf(m), background=(200, 100, 50))],
    'scale_out': lambda m: [m.geo.Scale(0.7, clip_boxes=False)],
    'rotate90': lambda m: [m.geo.Rotate(90)],
    'rotate180': lambda m: [m.geo.Rotate(180)],
    'rotate270': lambda m: [m.geo.Rotate(270)],
    'crop_pad': lambda m: [m.patch.CropPad(5, -7, 40, 60, box_filter=_bf(m))],
    'crop_pad_bg': lambda m: [m.patch.CropPad(-5, 3, 30, 80, clip_boxes=False, background=(1, 2, 3))],
    'crop': lambda m: [m.patch.Crop(3, 5, 7, 2, box_filter=_bf(m))],
    'pad': lambda m: [m.patch.Pad(4, 6, 8, 2, background=(9, 8, 7))],
    'patch_inf': lambda m: [m.patch.RandomPatchInf(m.patch.PatchCoordinateGenerator(must_match='h_ar', min_scale=0.4, max_scale=1.2,
                                                                                     min_aspect_ratio=0.6, max_aspect_ratio=1.6),
                                                   box_filter=_bf(m), image_validator=_iv(m), n_trials_max=4, prob=0.7)],
    'max_crop': lambda m: [m.patch.RandomMaxCropFixedAR(1.5, box_filter=_bf(m), image_validator=_iv(m), n_trials_max=3)],
    'pad_ar': lambda m: [m.patch.RandomPadFixedAR(0.75, background=(5, 6, 7))],
    'rgb2hsv': lambda m: [_hsv(m)],
    'hsv2rgb': lambda m: [_rgb(m)],
    'rgb2rgb': lambda m: [m.photo.ConvertColor('RGB', 'RGB')],
    'dtype': lambda m: [_f32(m), _u8(m)],
    'brightness': lambda m: [_f32(m), m.photo.Brightness(20.5), _u8(m)],
    'contrast': lambda m: [_f32(m), m.photo.Contrast(1.3), _u8(m)],
    'saturation': lambda m: [_hsv(m), _f32(m), m.photo.Saturation(1.4), _u8(m), _rgb(m)],
    'hue': lambda m: [_hsv(m), _f32(m), m.photo.Hue(-12.5), _u8(m), _rgb(m)],
    'channel_swap': lambda m: [m.photo.ChannelSwap((2, 0, 1))],
    'random_channel_swap': lambda m: [m.photo.RandomChannelSwap(prob=0.9)],
    'equalize': lambda m: [_hsv(m), m.photo.HistogramEqualization(), _rgb(m)],
    'equalize_rgb': lambda m: [m.photo.HistogramEqualization()],
    'random_equalize': lambda m: [_hsv(m), m.photo.RandomHistogramEqualization(prob=0.6), _rgb(m)],
}
SINGLE_SEED = 31


def _chain_equalize(m):
    return [m.photo.ConvertTo3Channels(), _hsv(m), m.photo.RandomHistogramEqualization(prob=0.5), _rgb(m), m.geo.Flip('horizontal'),
            m.geo.Translate(0.1, -0.05, box_filter=_bf(m)), m.patch.RandomPadFixedAR(1.0), m.geo.Resize(48, 48)]


def _chain_photometric(m):
    return [m.photo.ConvertTo3Channels(), _f32(m), m.photo.Brightness(-20), m.photo.Contrast(1.2), _u8(m),
            m.photo.RandomChannelSwap(prob=0.5), _hsv(m), m.photo.HistogramEqualization(), _f32(m), m.photo.Saturation(1.3),
            m.photo.Hue(10), _u8(m), m.photo.HistogramEqualization(), _rgb(m), m.geo.Rotate(90), m.patch.Crop(2, 3, 4, 1),
            m.patch.RandomMaxCropFixedAR(1.25), m.geo.Resize(40, 50)]


def _chain_patch(m):
    bg = (50, 60, 70)
    pcg = m.patch.PatchCoordinateGenerator(must_match='w_ar', min_scale=0.5, max_scale=1.0, min_aspect_ratio=0.7, max_aspect_ratio=1.4)
    # ConvertColor before the equalisation: the reference's equalises its input in place, which would change a 3-channel image of
    # the in-memory dataset for the next epoch
    return [m.photo.ConvertTo3Channels(), _rgb(m), m.photo.RandomHistogramEqualization(prob=0.5), _hsv(m),
            m.patch.Pad(5, 3, 2, 8, background=bg),
            m.patch.RandomPatchInf(pcg, box_filter=_bf(m), image_validator=_iv(m), n_trials_max=3, prob=0.8, background=bg),
            m.geo.Flip('vertical'), m.geo.Resize(36, 44, box_filter=m.valid.BoxFilter(check_overlap=False, check_min_area=False))]


# name: (transformations, dataset, labels dtype, seed, batches); 10 images in batches of 4: a short last batch, then a reshuffle
CHAINS = {
    'equalize': (_chain_equalize, ds.variable_dataset, 'int', 41, 4),
    'photometric': (_chain_photometric, ds.variable_dataset, 'float', 42, 4),
    'patch': (_chain_patch, ds.variable_dataset, 'int', 43, 4),
}
