/*
 * bdev_oimgpu_rpc.c — construct_oimgpu_bdev / delete_oimgpu_bdev.  Parameters, validation and error replies are
 * those of construct_malloc_bdev / delete_malloc_bdev (S/lib/bdev/malloc/bdev_malloc_rpc.c:63-106,144-170), so a
 * client that builds Malloc disks builds HBM disks by changing the method name.
 */
#include "spdk/stdinc.h"

#include "spdk/bdev.h"
#include "spdk/json.h"
#include "spdk/jsonrpc.h"
#include "spdk/rpc.h"
#include "spdk/string.h"
#include "spdk/util.h"
#include "spdk/uuid.h"

#include "bdev_oimgpu.h"

struct rpc_construct_oimgpu {
	char		*name;
	char		*uuid;
	uint64_t	num_blocks;
	uint32_t	block_size;
};

static const struct spdk_json_object_decoder rpc_construct_oimgpu_decoders[] = {
	{"name", offsetof(struct rpc_construct_oimgpu, name), spdk_json_decode_string, true},
	{"uuid", offsetof(struct rpc_construct_oimgpu, uuid), spdk_json_decode_string, true},
	{"num_blocks", offsetof(struct rpc_construct_oimgpu, num_blocks), spdk_json_decode_uint64},
	{"block_size", offsetof(struct rpc_construct_oimgpu, block_size), spdk_json_decode_uint32},
};

static void
spdk_rpc_construct_oimgpu_bdev(struct spdk_jsonrpc_request *request, const struct spdk_json_val *params)
{
	struct rpc_construct_oimgpu req = {};
	struct spdk_uuid uuid;
	struct spdk_bdev *bdev = NULL;
	struct spdk_json_write_ctx *w;

	if (spdk_json_decode_object(params, rpc_construct_oimgpu_decoders,
				    SPDK_COUNTOF(rpc_construct_oimgpu_decoders), &req) == 0 &&
	    (!req.uuid || spdk_uuid_parse(&uuid, req.uuid) == 0)) {
		bdev = create_oimgpu_disk(req.name, req.uuid ? &uuid : NULL, req.num_blocks, req.block_size);
	}
	free(req.name);
	free(req.uuid);
	if (!bdev) {
		spdk_jsonrpc_send_error_response(request, SPDK_JSONRPC_ERROR_INVALID_PARAMS, "Invalid parameters");
		return;
	}
	w = spdk_jsonrpc_begin_result(request);
	if (w) {
		spdk_json_write_string(w, spdk_bdev_get_name(bdev));
		spdk_jsonrpc_end_result(request, w);
	}
}
SPDK_RPC_REGISTER("construct_oimgpu_bdev", spdk_rpc_construct_oimgpu_bdev, SPDK_RPC_RUNTIME)

struct rpc_delete_oimgpu {
	char *name;
};

static const struct spdk_json_object_decoder rpc_delete_oimgpu_decoders[] = {
	{"name", offsetof(struct rpc_delete_oimgpu, name), spdk_json_decode_string},
};

static void
rpc_delete_oimgpu_bdev_done(void *cb_arg, int bdeverrno)
{
	struct spdk_jsonrpc_request *request = cb_arg;
	struct spdk_json_write_ctx *w = spdk_jsonrpc_begin_result(request);

	if (w) {
		spdk_json_write_bool(w, bdeverrno == 0);
		spdk_jsonrpc_end_result(request, w);
	}
}

static void
spdk_rpc_delete_oimgpu_bdev(struct spdk_jsonrpc_request *request, const struct spdk_json_val *params)
{
	struct rpc_delete_oimgpu req = {};
	struct spdk_bdev *bdev;
	int rc;

	if (spdk_json_decode_object(params, rpc_delete_oimgpu_decoders,
				    SPDK_COUNTOF(rpc_delete_oimgpu_decoders), &req)) {
		rc = -EINVAL;
	} else if ((bdev = spdk_bdev_get_by_name(req.name)) == NULL) {
		rc = -ENODEV;
	} else {
		delete_oimgpu_disk(bdev, rpc_delete_oimgpu_bdev_done, request);
		free(req.name);
		return;
	}
	free(req.name);
	spdk_jsonrpc_send_error_response(request, SPDK_JSONRPC_ERROR_INVALID_PARAMS, spdk_strerror(-rc));
}
SPDK_RPC_REGISTER("delete_oimgpu_bdev", spdk_rpc_delete_oimgpu_bdev, SPDK_RPC_RUNTIME)
