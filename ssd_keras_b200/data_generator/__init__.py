"""The data pipeline on the device (SURVEY.md section 8f): ``DataGenerator`` (``parse_csv``, ``parse_xml``, ``parse_json`` and
``generate``) with the original SSD, SSD7 (constant input size), variable-input-size and satellite augmentation chains, or custom
chains of the op modules' classes, drawn on the host and run on the device, batch assembly for the encoder, box and image transforms of the geometric and photometric ops,
and the inverse-transform helper.  HDF5 datasets and image decoding on the device stay out of scope."""
