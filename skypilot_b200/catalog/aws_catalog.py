"""AWS catalog: the function table of sky/catalog/aws_catalog.py, served
from the GPU-resident store (see _cloud_catalog.CloudCatalog). Like the
reference's `_get_df()`, the store holds the catalog after the account's zone
mapping (store.apply_az_mapping): zone names where a mapping was loaded, the
catalog's zone IDs otherwise."""
from skypilot_b200.catalog import _cloud_catalog

_impl = _cloud_catalog.CloudCatalog('aws', supports_zones=True)

instance_type_exists = _impl.instance_type_exists
validate_region_zone = _impl.validate_region_zone
get_hourly_cost = _impl.get_hourly_cost
get_vcpus_mem_from_instance_type = _impl.get_vcpus_mem_from_instance_type
get_default_instance_type = _impl.get_default_instance_type
get_accelerators_from_instance_type = _impl.get_accelerators_from_instance_type
get_arch_from_instance_type = _impl.get_arch_from_instance_type
get_local_disk_from_instance_type = _impl.get_local_disk_from_instance_type
get_instance_type_for_accelerator = _impl.get_instance_type_for_accelerator
get_region_zones_for_instance_type = _impl.get_region_zones_for_instance_type
list_accelerators = _impl.list_accelerators
get_image_id_from_tag = _impl.get_image_id_from_tag
is_image_tag_valid = _impl.is_image_tag_valid
