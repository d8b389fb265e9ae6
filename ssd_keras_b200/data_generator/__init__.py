"""The data pipeline on the device (SURVEY.md section 8f): ``DataGenerator.generate`` with the original SSD augmentation chain
(``data_augmentation_chain_original_ssd``) drawn on the host and run on the device, batch assembly for the encoder, box and
image transforms of the geometric and photometric ops, and the inverse-transform helper.  Dataset parsers, HDF5 datasets and
image decoding on the device stay out of scope."""
