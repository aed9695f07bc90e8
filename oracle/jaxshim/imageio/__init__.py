"""Import stub: nerfies/image_utils.py imports imageio; the data path recorded by
oracle/make_golden_data.py decodes images with cv2 and never calls it."""
