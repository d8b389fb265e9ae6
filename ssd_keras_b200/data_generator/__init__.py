"""The hand-off between the reference's data pipeline and the hot path (SURVEY.md section 8f): batch assembly for the encoder,
box and image transforms of the geometric ops on the device and the inverse-transform helper.  Dataset parsing, image
decoding and photometric augmentation stay out of scope."""
