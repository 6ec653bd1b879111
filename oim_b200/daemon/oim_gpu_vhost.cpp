/*
 * oim-gpu-vhost — drop-in for the SPDK `vhost` daemon behind intel/oim's unmodified Go binaries
 * (SURVEY.md §8(b) B1).  Speaks the JSON-RPC 2.0 dialect pkg/spdk/client.go:121-212 expects over an
 * AF_UNIX stream socket and maps the twelve methods pkg/spdk/spdk.go:47-286 issues onto the C ABI of
 * liboimgpu (include/oimgpu.h).  Wire behaviour follows the reference server:
 *   framing / errors     S/lib/jsonrpc/jsonrpc_server.c:54-101,240-341  (newline after every reply,
 *                        "id" echoed verbatim, notifications get no reply, parse error closes)
 *   bdev methods         S/lib/bdev/rpc/bdev_rpc.c:216-433, S/lib/bdev/malloc/bdev_malloc_rpc.c:63-106,
 *                        S/lib/bdev/rbd/bdev_rbd_rpc.c:102-148
 *   vhost methods        S/lib/vhost/vhost_rpc.c:65-478
 * and is pinned against the reference's own server running in-process (tests/test_rpc_daemon.py).  Four methods are the
 * project's own, for mirrored bdevs: construct_mirror_bdev, export_bdev_store, check_mirror_bdev and
 * replace_mirror_replica (INTEGRATION.md 3c); two more, save_bdev_image and load_bdev_image, move any bdev's bytes to
 * and from a sparse image file, and three, enable_bdev_image_tracking, save_bdev_image_delta and
 * apply_bdev_image_delta, move only what changed since the last image (INTEGRATION.md 3d).
 *
 * CLI as S/app/vhost/vhost.c:43-48 + S/lib/event/app.c:826-960:
 *   -S <dir> vhost socket directory   -r <path> RPC socket (default /var/tmp/spdk.sock)
 *   -f <pidfile>   -m <core mask>   -s <MB> / -R accepted and ignored   --gpus 0,1,..  GPUs to use
 *
 * Control plane only: no request data passes through this process.
 */
#include <cerrno>
#include <csignal>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include <fcntl.h>
#include <poll.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <sys/un.h>
#include <unistd.h>

#include <linux/nbd.h>
#include <sys/ioctl.h>
#include <memory>
#include <thread>

#include "oimgpu.h"
#include "vhost_user.h"

/* ---- a small JSON value (parse + the subset of writing the replies need) ------------------------ */

struct Json {
	enum Type { Null, Bool, Num, Str, Arr, Obj } type = Null;
	bool b = false;
	std::string raw;	/* number text or decoded string */
	std::vector<Json> arr;
	std::vector<std::pair<std::string, Json>> obj;

	const Json *get(const char *key) const
	{
		for (auto &kv : obj) if (kv.first == key) return &kv.second;
		return nullptr;
	}
};

struct Parser {
	const char *p, *end;
	bool incomplete = false;

	void ws() { while (p < end && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r')) p++; }

	bool string(std::string &out)
	{
		if (p >= end) { incomplete = true; return false; }
		if (*p != '"') return false;
		p++;
		while (true) {
			if (p >= end) { incomplete = true; return false; }
			char c = *p++;
			if (c == '"') return true;
			if ((unsigned char)c < 0x20) return false;
			if (c != '\\') { out += c; continue; }
			if (p >= end) { incomplete = true; return false; }
			char e = *p++;
			switch (e) {
			case '"': out += '"'; break;
			case '\\': out += '\\'; break;
			case '/': out += '/'; break;
			case 'b': out += '\b'; break;
			case 'f': out += '\f'; break;
			case 'n': out += '\n'; break;
			case 'r': out += '\r'; break;
			case 't': out += '\t'; break;
			case 'u': {
				if (end - p < 4) { incomplete = true; return false; }
				unsigned v = 0;
				for (int i = 0; i < 4; i++) {
					char h = *p++;
					v <<= 4;
					if (h >= '0' && h <= '9') v |= h - '0';
					else if (h >= 'a' && h <= 'f') v |= h - 'a' + 10;
					else if (h >= 'A' && h <= 'F') v |= h - 'A' + 10;
					else return false;
				}
				if (v < 0x80) out += (char)v;
				else if (v < 0x800) { out += (char)(0xC0 | v >> 6); out += (char)(0x80 | (v & 0x3F)); }
				else { out += (char)(0xE0 | v >> 12); out += (char)(0x80 | ((v >> 6) & 0x3F)); out += (char)(0x80 | (v & 0x3F)); }
				break;
			}
			default: return false;
			}
		}
	}

	bool value(Json &v, int depth = 0)
	{
		if (depth > 32) return false;
		ws();
		if (p >= end) { incomplete = true; return false; }
		char c = *p;
		if (c == '{') {
			v.type = Json::Obj;
			p++;
			ws();
			if (p < end && *p == '}') { p++; return true; }
			while (true) {
				ws();
				std::string k;
				if (!string(k)) return false;
				ws();
				if (p >= end) { incomplete = true; return false; }
				if (*p++ != ':') return false;
				Json child;
				if (!value(child, depth + 1)) return false;
				v.obj.emplace_back(std::move(k), std::move(child));
				ws();
				if (p >= end) { incomplete = true; return false; }
				if (*p == ',') { p++; continue; }
				if (*p == '}') { p++; return true; }
				return false;
			}
		}
		if (c == '[') {
			v.type = Json::Arr;
			p++;
			ws();
			if (p < end && *p == ']') { p++; return true; }
			while (true) {
				Json child;
				if (!value(child, depth + 1)) return false;
				v.arr.push_back(std::move(child));
				ws();
				if (p >= end) { incomplete = true; return false; }
				if (*p == ',') { p++; continue; }
				if (*p == ']') { p++; return true; }
				return false;
			}
		}
		if (c == '"') { v.type = Json::Str; return string(v.raw); }
		auto lit = [&](const char *s, Json::Type t, bool b) {
			size_t n = strlen(s);
			if ((size_t)(end - p) < n) {
				if (strncmp(p, s, end - p) == 0) incomplete = true;
				return false;
			}
			if (strncmp(p, s, n)) return false;
			p += n; v.type = t; v.b = b;
			return true;
		};
		if (c == 't') return lit("true", Json::Bool, true);
		if (c == 'f') return lit("false", Json::Bool, false);
		if (c == 'n') return lit("null", Json::Null, false);
		if (c == '-' || (c >= '0' && c <= '9')) {
			const char *s = p;
			if (*p == '-') p++;
			while (p < end && ((*p >= '0' && *p <= '9') || *p == '.' || *p == 'e' || *p == 'E' || *p == '+' || *p == '-')) p++;
			if (p == end) { incomplete = true; return false; }	/* the number may continue in the next read */
			v.type = Json::Num;
			v.raw.assign(s, p - s);
			return v.raw != "-";
		}
		return false;
	}
};

static std::string jstr(const std::string &s)
{
	std::string o = "\"";
	for (unsigned char c : s) {
		switch (c) {
		case '"': o += "\\\""; break;
		case '\\': o += "\\\\"; break;
		case '\b': o += "\\b"; break;
		case '\f': o += "\\f"; break;
		case '\n': o += "\\n"; break;
		case '\r': o += "\\r"; break;
		case '\t': o += "\\t"; break;
		default:
			if (c < 0x20) { char b[8]; snprintf(b, sizeof(b), "\\u%04x", c); o += b; }
			else o += (char)c;
		}
	}
	return o + "\"";
}

/* ---- parameter decoding with spdk_json_decode_object's rules (S/lib/json/json_util.c:302-370):
 *      unknown key, duplicate key, wrong type or missing mandatory key => failure --------------- */

struct Field { const char *name; Json::Type type; bool optional; const Json **out; };

static bool decode(const Json *params, std::vector<Field> fields)
{
	if (!params || params->type != Json::Obj) return false;
	std::vector<bool> seen(fields.size(), false);
	bool ok = true;
	for (auto &kv : params->obj) {
		bool found = false;
		for (size_t i = 0; i < fields.size(); i++) {
			if (kv.first != fields[i].name) continue;
			found = true;
			if (seen[i] || kv.second.type != fields[i].type) ok = false;
			else *fields[i].out = &kv.second;
			seen[i] = true;
		}
		if (!found) ok = false;
	}
	for (size_t i = 0; i < fields.size(); i++) if (!seen[i] && !fields[i].optional) ok = false;
	return ok;
}

/* spdk_json_number_to_uint64 / int32 for plain integers (no fraction, no exponent) */
static bool to_u64(const Json *j, uint64_t *out)
{
	if (!j || j->type != Json::Num || j->raw.empty() || j->raw[0] == '-') return false;
	for (char c : j->raw) if (c < '0' || c > '9') return false;
	errno = 0;
	char *e = nullptr;
	unsigned long long v = strtoull(j->raw.c_str(), &e, 10);
	if (errno || *e) return false;
	*out = v;
	return true;
}
static bool to_i32(const Json *j, int32_t *out)
{
	if (!j || j->type != Json::Num) return false;
	const char *s = j->raw.c_str();
	for (const char *c = s + (*s == '-'); *c; c++) if (*c < '0' || *c > '9') return false;
	errno = 0;
	long long v = strtoll(s, nullptr, 10);
	if (errno || v < INT32_MIN || v > INT32_MAX) return false;
	*out = (int32_t)v;
	return true;
}

/* ---- replies -------------------------------------------------------------------------------------- */

struct Reply { bool has = false; std::string body; };

static std::string id_text(const Json *id)
{
	if (!id || id->type == Json::Null) return "null";
	return id->type == Json::Str ? jstr(id->raw) : id->raw;
}
static Reply result(const Json *id, const std::string &r)
{
	Reply rp;
	if (!id || id->type == Json::Null) return rp;	/* notification: no response (jsonrpc_server.c:296-300) */
	rp.has = true;
	rp.body = "{\"jsonrpc\":\"2.0\",\"id\":" + id_text(id) + ",\"result\":" + r + "}\n";
	return rp;
}
static Reply error(const Json *id, int code, const std::string &msg)
{
	Reply rp;
	rp.has = true;
	rp.body = "{\"jsonrpc\":\"2.0\",\"id\":" + id_text(id) + ",\"error\":{\"code\":" + std::to_string(code) +
		  ",\"message\":" + jstr(msg) + "}}\n";
	return rp;
}
enum { E_PARSE = -32700, E_INVALID_REQUEST = -32600, E_METHOD_NOT_FOUND = -32601, E_INVALID_PARAMS = -32602, E_INTERNAL = -32603 };

static std::string strerr(int rc) { return strerror(rc < 0 ? -rc : rc); }

/* ---- the twelve methods ---------------------------------------------------------------------------- */

static std::string bdev_json(const oimgpu_bdev_info &b)
{
	/* spdk_rpc_dump_bdev_info (bdev_rpc.c:216-300) for a bdev without QoS, aliases or driver info */
	std::string s = "{\"name\":" + jstr(b.name) + ",\"aliases\":[],\"product_name\":" + jstr(b.product_name) +
			",\"block_size\":" + std::to_string(b.block_size) + ",\"num_blocks\":" + std::to_string(b.num_blocks);
	if (b.uuid[0]) s += ",\"uuid\":" + jstr(b.uuid);
	s += ",\"assigned_rate_limits\":{\"rw_ios_per_sec\":0,\"rw_mbytes_per_sec\":0,\"r_mbytes_per_sec\":0,\"w_mbytes_per_sec\":0}";
	s += std::string(",\"claimed\":") + (b.claimed ? "true" : "false");
	s += ",\"supported_io_types\":{\"read\":true,\"write\":true,\"unmap\":true,\"write_zeroes\":true,\"flush\":true,"
	     "\"reset\":true,\"nvme_admin\":false,\"nvme_io\":false},\"driver_specific\":{";
	if (b.replicas > 1) {
		/* a mirror (a project bdev: the reference has none) says where its replicas are */
		s += "\"mirror\":{\"replicas\":[";
		for (uint32_t r = 0; r < b.replicas; r++) {
			int dev = 0, imported = 0;
			oimgpu_bdev_replica_info(b.name, (int)r, &dev, &imported);
			s += std::string(r ? "," : "") + "{\"gpu\":" + std::to_string(dev) + ",\"imported\":" + (imported ? "true" : "false") + "}";
		}
		s += "]}";
	}
	return s + "}}";
}

static std::string base64_encode(const uint8_t *p, size_t n)
{
	static const char tbl[] = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
	std::string o;
	o.reserve((n + 2) / 3 * 4);
	for (size_t i = 0; i < n; i += 3) {
		const uint32_t v = (uint32_t)p[i] << 16 | (i + 1 < n ? (uint32_t)p[i + 1] << 8 : 0) | (i + 2 < n ? p[i + 2] : 0);
		o += tbl[v >> 18]; o += tbl[(v >> 12) & 63];
		o += i + 1 < n ? tbl[(v >> 6) & 63] : '=';
		o += i + 2 < n ? tbl[v & 63] : '=';
	}
	return o;
}

/* strict RFC 4648 base64 (padded, no whitespace); false on anything else */
static bool base64_decode(const std::string &s, std::string *out)
{
	if (s.size() % 4) return false;
	out->clear();
	for (size_t i = 0; i < s.size(); i += 4) {
		uint32_t v = 0;
		int pad = 0;
		for (int k = 0; k < 4; k++) {
			const char c = s[i + k];
			int d;
			if (c >= 'A' && c <= 'Z') d = c - 'A';
			else if (c >= 'a' && c <= 'z') d = c - 'a' + 26;
			else if (c >= '0' && c <= '9') d = c - '0' + 52;
			else if (c == '+') d = 62;
			else if (c == '/') d = 63;
			else if (c == '=' && i + 4 == s.size() && k >= 2) { d = 0; pad++; }
			else return false;
			if (pad && c != '=') return false;	/* nothing may follow padding */
			v = v << 6 | (uint32_t)d;
		}
		*out += (char)(v >> 16);
		if (pad < 2) *out += (char)(v >> 8 & 0xFF);
		if (pad < 1) *out += (char)(v & 0xFF);
	}
	return true;
}

static std::string ctrlr_json(const oimgpu_ctrlr_info &c)
{
	/* _spdk_rpc_get_vhost_controller (vhost_rpc.c:378-402) + spdk_vhost_scsi_dump_info_json (vhost_scsi.c:1410-1456) */
	std::string s = "{\"ctrlr\":" + jstr(c.ctrlr) + ",\"cpumask\":" + jstr(c.cpumask) +
			",\"delay_base_us\":" + std::to_string(c.delay_base_us) + ",\"iops_threshold\":" + std::to_string(c.iops_threshold) +
			",\"socket\":" + jstr(c.socket) + ",\"backend_specific\":{\"scsi\":[";
	for (uint32_t i = 0; i < c.ntargets; i++) {
		const oimgpu_target_info &t = c.targets[i];
		if (i) s += ",";
		s += "{\"scsi_dev_num\":" + std::to_string(t.scsi_dev_num) + ",\"id\":" + std::to_string(t.id) +
		     ",\"target_name\":" + jstr(t.target_name) + ",\"luns\":[{\"id\":" + std::to_string(t.lun_id) +
		     ",\"bdev_name\":" + jstr(t.bdev_name) + "}]}";
	}
	return s + "]}}";
}

/* an exported bdev: /dev/nbdX <- kernel end of a socketpair; our end is served by oimgpu_nbd_serve */
struct NbdDisk {
	std::string dev, bdev;
	int dev_fd = -1, kernel_fd = -1, our_fd = -1;
	std::thread serve, doit;
};
static std::vector<std::unique_ptr<NbdDisk>> g_nbd;

/* spdk_nbd_start + spdk_nbd_enable_kernel + spdk_nbd_start_complete (S/lib/nbd/nbd.c:867-1060): hand one end
 * of a socketpair to the kernel NBD device, describe the disk, let a thread sit in NBD_DO_IT, serve the other
 * end.  Returns 0 or -errno; every failure becomes "Invalid parameters" on the wire (nbd_rpc.c:63-70). */
static int nbd_start(const std::string &bdev, const std::string &dev)
{
	oimgpu_bdev_info info;
	if (oimgpu_bdev_get(bdev.c_str(), &info) != 0) return -EINVAL;
	auto d = std::make_unique<NbdDisk>();
	d->dev = dev;
	d->bdev = bdev;
	int sp[2];
	if (socketpair(AF_UNIX, SOCK_STREAM, 0, sp) != 0) return -errno;
	d->our_fd = sp[0];
	d->kernel_fd = sp[1];
	auto fail = [&](int rc) {
		close(d->our_fd);
		close(d->kernel_fd);
		if (d->dev_fd >= 0) close(d->dev_fd);
		return rc;
	};
	d->dev_fd = open(dev.c_str(), O_RDWR);
	if (d->dev_fd < 0) return fail(-errno);
	int rc = -1;
	for (int tries = 0; tries < 1000; tries++) {	/* NBD_BUSY_WAITING_MS: the kernel may still be tearing a previous user down */
		rc = ioctl(d->dev_fd, NBD_SET_SOCK, d->kernel_fd);
		if (rc == 0 || errno != EBUSY) break;
		usleep(1000);
	}
	if (rc != 0) return fail(-errno);
	if (ioctl(d->dev_fd, NBD_SET_BLKSIZE, (unsigned long)info.block_size) != 0 ||
	    ioctl(d->dev_fd, NBD_SET_SIZE_BLOCKS, (unsigned long)info.num_blocks) != 0 ||
	    ioctl(d->dev_fd, NBD_SET_FLAGS, (unsigned long)NBD_FLAG_SEND_TRIM) != 0) {
		rc = -errno;
		ioctl(d->dev_fd, NBD_CLEAR_SOCK);
		return fail(rc);
	}
	NbdDisk *p = d.get();
	d->doit = std::thread([p] { ioctl(p->dev_fd, NBD_DO_IT); });	/* blocks in the kernel until our end closes */
	d->serve = std::thread([p] { oimgpu_nbd_serve(p->bdev.c_str(), p->our_fd); });
	g_nbd.push_back(std::move(d));
	return 0;
}

/* spdk_nbd_stop / _nbd_stop (nbd.c:346-395) */
static void nbd_stop(NbdDisk &d)
{
	shutdown(d.our_fd, SHUT_RDWR);
	if (d.serve.joinable()) d.serve.join();
	close(d.our_fd);
	close(d.kernel_fd);
	ioctl(d.dev_fd, NBD_CLEAR_QUE);
	ioctl(d.dev_fd, NBD_CLEAR_SOCK);
	if (d.doit.joinable()) d.doit.join();
	close(d.dev_fd);
}
static uint64_t g_rbd_default_size = 8ull << 30;
static bool g_serve_vhost_user = true;

static Reply dispatch(const std::string &method, const Json *params, const Json *id)
{
	const Json *a = nullptr, *b = nullptr, *c = nullptr, *d = nullptr, *e = nullptr, *f = nullptr;
	const Reply bad = error(id, E_INVALID_PARAMS, "Invalid parameters");

	if (method == "get_bdevs") {
		if (params && !decode(params, {{"name", Json::Str, true, &a}})) return bad;
		std::string out = "[";
		if (a) {
			oimgpu_bdev_info info;
			if (oimgpu_bdev_get(a->raw.c_str(), &info) != 0) return bad;
			out += bdev_json(info);
		} else {
			int n = oimgpu_bdev_list(nullptr, 0);
			std::vector<oimgpu_bdev_info> v(n > 0 ? n : 1);
			n = oimgpu_bdev_list(v.data(), n);
			for (int i = 0; i < n; i++) out += (i ? "," : "") + bdev_json(v[i]);
		}
		return result(id, out + "]");
	}
	if (method == "get_bdevs_iostat") {
		/* S/lib/bdev/rpc/bdev_rpc.c:50-205.  tick_rate is the GPU's global timer (1 GHz); the *_latency_ticks are summed
		 * per request by the mover warps (pass fetched -> data moved), see include/oimgpu.h struct oimgpu_iostat. */
		if (params && !decode(params, {{"name", Json::Str, true, &a}})) return bad;
		std::vector<std::string> names;
		if (a) {
			oimgpu_bdev_info info;
			if (oimgpu_bdev_get(a->raw.c_str(), &info) != 0) return bad;
			names.push_back(info.name);
		} else {
			int n = oimgpu_bdev_list(nullptr, 0);
			std::vector<oimgpu_bdev_info> v(n > 0 ? n : 1);
			n = oimgpu_bdev_list(v.data(), n);
			for (int i = 0; i < n; i++) names.push_back(v[i].name);
		}
		std::string out = "[{\"tick_rate\":1000000000}";
		for (auto &nm : names) {
			oimgpu_iostat st;
			if (oimgpu_bdev_iostat(nm.c_str(), &st) != 0) continue;
			out += ",{\"name\":" + jstr(nm) + ",\"bytes_read\":" + std::to_string(st.bytes_read) +
			       ",\"num_read_ops\":" + std::to_string(st.num_read_ops) + ",\"bytes_written\":" + std::to_string(st.bytes_written) +
			       ",\"num_write_ops\":" + std::to_string(st.num_write_ops) + ",\"bytes_unmapped\":" + std::to_string(st.bytes_unmapped) +
			       ",\"num_unmap_ops\":" + std::to_string(st.num_unmap_ops) +
			       ",\"read_latency_ticks\":" + std::to_string(st.read_latency_ns) + ",\"write_latency_ticks\":" +
			       std::to_string(st.write_latency_ns) + ",\"unmap_latency_ticks\":" + std::to_string(st.unmap_latency_ns) + "}";
		}
		return result(id, out + "]");
	}
	if (method == "enable_bdev_histogram") {
		/* S/lib/bdev/rpc/bdev_rpc.c:607-671 */
		if (!decode(params, {{"name", Json::Str, false, &a}, {"enable", Json::Bool, false, &b}})) return error(id, E_INVALID_PARAMS, strerr(EINVAL));
		int rc = oimgpu_bdev_histogram_enable(a->raw.c_str(), b->b ? 1 : 0);
		if (rc == -ENODEV) return error(id, E_INVALID_PARAMS, strerr(ENODEV));
		return result(id, rc == 0 ? "true" : "false");
	}
	if (method == "get_bdev_histogram") {
		/* bdev_rpc.c:675-790: {"histogram": base64 of the bucket array, "bucket_shift": 7, "tsc_rate": ticks per second} */
		if (!decode(params, {{"name", Json::Str, false, &a}})) return error(id, E_INVALID_PARAMS, strerr(EINVAL));
		std::vector<uint64_t> buckets(OIMGPU_HISTOGRAM_BUCKETS);
		int rc = oimgpu_bdev_histogram_get(a->raw.c_str(), buckets.data());
		if (rc == -ENODEV) return error(id, E_INVALID_PARAMS, strerr(ENODEV));
		if (rc < 0) return error(id, E_INTERNAL, strerr(rc));
		const std::string b64 = base64_encode((const uint8_t *)buckets.data(), buckets.size() * sizeof(uint64_t));
		return result(id, "{\"histogram\":\"" + b64 + "\",\"bucket_shift\":7,\"tsc_rate\":1000000000}");
	}
	if (method == "construct_malloc_bdev") {
		uint64_t nb = 0, bs = 0;
		if (!decode(params, {{"name", Json::Str, true, &a}, {"uuid", Json::Str, true, &b},
				     {"num_blocks", Json::Num, false, &c}, {"block_size", Json::Num, false, &d}})) return bad;
		if (!to_u64(c, &nb) || !to_u64(d, &bs) || bs > UINT32_MAX) return bad;
		char name[64];
		int rc = oimgpu_bdev_create_malloc(a ? a->raw.c_str() : nullptr, b ? b->raw.c_str() : nullptr, nb, (uint32_t)bs, -1, name, sizeof(name));
		if (rc != 0) return bad;
		return result(id, jstr(name));
	}
	if (method == "construct_rbd_bdev") {
		/* bdev_rbd_rpc.c:64-148: pool_name, rbd_name, block_size mandatory; name, user_id, config optional */
		uint64_t bs = 0;
		if (!decode(params, {{"name", Json::Str, true, &a}, {"user_id", Json::Str, true, &b}, {"pool_name", Json::Str, false, &c},
				     {"rbd_name", Json::Str, false, &d}, {"block_size", Json::Num, false, &e}, {"config", Json::Obj, true, &f}})) return bad;
		if (!to_u64(e, &bs) || bs > UINT32_MAX) return bad;
		if (f) for (auto &kv : f->obj) if (kv.second.type != Json::Str) return bad;	/* config: string -> string */
		char name[64];
		int rc = oimgpu_bdev_create_rbd(a ? a->raw.c_str() : nullptr, c->raw.c_str(), d->raw.c_str(), b ? b->raw.c_str() : nullptr,
						(uint32_t)bs, g_rbd_default_size, -1, name, sizeof(name));
		if (rc != 0) return bad;
		return result(id, jstr(name));
	}
	if (method == "construct_mirror_bdev") {
		/* project method (the reference has no mirror, SURVEY.md 8(c)), shaped and answered like construct_malloc_bdev:
		 * `replicas` in-process replicas placed by the library's rule, or replica 0 here and `remote_replicas` the
		 * stores of other processes (base64 CUDA IPC handles, as export_bdev_store gives them) */
		uint64_t nb = 0, bs = 0, nrep = 0;
		if (!decode(params, {{"name", Json::Str, true, &a}, {"uuid", Json::Str, true, &b}, {"num_blocks", Json::Num, false, &c},
				     {"block_size", Json::Num, false, &d}, {"replicas", Json::Num, true, &e}, {"remote_replicas", Json::Arr, true, &f}}))
			return bad;
		if (!to_u64(c, &nb) || !to_u64(d, &bs) || bs > UINT32_MAX || !e == !f) return bad;
		const char *nm = a ? a->raw.c_str() : nullptr, *uuid = b ? b->raw.c_str() : nullptr;
		char name[64];
		int rc;
		if (e) {
			if (!to_u64(e, &nrep) || nrep < 2 || nrep > 4) return bad;
			rc = oimgpu_bdev_create_mirror_uuid(nm, uuid, nb, (uint32_t)bs, nullptr, (int)nrep, name, sizeof(name));
		} else {
			if (f->arr.empty() || f->arr.size() > 3) return bad;
			std::string handles, h;
			for (auto &x : f->arr) {
				if (x.type != Json::Str || !base64_decode(x.raw, &h) || h.size() != OIMGPU_IPC_HANDLE_BYTES) return bad;
				handles += h;
			}
			rc = oimgpu_bdev_create_mirror_remote_uuid(nm, uuid, nb, (uint32_t)bs, -1, handles.data(), (int)f->arr.size(),
								   name, sizeof(name));
		}
		if (rc != 0) return bad;
		return result(id, jstr(name));
	}
	if (method == "export_bdev_store") {
		/* the CUDA IPC handle of one replica's store, for another process's construct_mirror_bdev {remote_replicas}.
		 * The bdev must outlive every mirror built on the handle: delete the importing mirror first. */
		int32_t rep = 0;
		if (!decode(params, {{"name", Json::Str, false, &a}, {"replica", Json::Num, true, &b}}) || (b && !to_i32(b, &rep)))
			return error(id, E_INVALID_PARAMS, strerr(EINVAL));
		uint8_t h[OIMGPU_IPC_HANDLE_BYTES];
		int rc = oimgpu_bdev_export_store(a->raw.c_str(), rep, h);
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		return result(id, "\"" + base64_encode(h, sizeof(h)) + "\"");
	}
	if (method == "check_mirror_bdev") {
		/* compare every replica with replica 0 (and copy replica 0 over the blocks that differ, with repair): md RAID1's
		 * check / repair.  At most kMaxRanges runs of differing blocks are listed; mismatched_blocks counts them all. */
		constexpr uint32_t kMaxRanges = 64;
		uint64_t off = 0, n = 0;
		if (!decode(params, {{"name", Json::Str, false, &a}, {"offset_blocks", Json::Num, true, &b}, {"num_blocks", Json::Num, true, &c},
				     {"repair", Json::Bool, true, &d}}) || (b && !to_u64(b, &off)) || (c && !to_u64(c, &n)))
			return bad;
		oimgpu_bdev_info info;
		int rc = oimgpu_bdev_get(a->raw.c_str(), &info);
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		if (!c) n = off <= info.num_blocks ? info.num_blocks - off : 0;
		uint64_t ranges[2 * kMaxRanges];
		oimgpu_mirror_check res;
		rc = oimgpu_bdev_mirror_check(a->raw.c_str(), off, n, d && d->b, ranges, kMaxRanges, &res);
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		std::string out = "{\"name\":" + jstr(info.name) + ",\"replicas\":" + std::to_string(info.replicas) +
				  ",\"offset_blocks\":" + std::to_string(off) + ",\"num_blocks\":" + std::to_string(n) +
				  ",\"mismatched_blocks\":" + std::to_string(res.mismatched_blocks) +
				  ",\"repaired_blocks\":" + std::to_string(res.repaired_blocks) + ",\"mismatches\":[";
		for (uint32_t k = 0; k < res.nranges; k++) {
			out += std::string(k ? "," : "") + "{\"offset_blocks\":" + std::to_string(ranges[2 * k]) +
			       ",\"num_blocks\":" + std::to_string(ranges[2 * k + 1]) + "}";
		}
		return result(id, out + "],\"truncated\":" + (res.truncated ? "true" : "false") + "}");
	}
	if (method == "replace_mirror_replica") {
		/* move an imported replica to the store behind `remote_replica` (a base64 handle, as export_bdev_store gives it):
		 * replica 0 is copied into it with the sessions held, and the old exporter may delete its bdev afterwards */
		int32_t rep = 0;
		std::string h;
		if (!decode(params, {{"name", Json::Str, false, &a}, {"replica", Json::Num, false, &b}, {"remote_replica", Json::Str, false, &c}}) ||
		    !to_i32(b, &rep) || !base64_decode(c->raw, &h) || h.size() != OIMGPU_IPC_HANDLE_BYTES)
			return bad;
		int rc = oimgpu_bdev_mirror_replace_remote(a->raw.c_str(), rep, h.data());
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		return result(id, "true");
	}
	if (method == "save_bdev_image" || method == "load_bdev_image") {
		/* a bdev's bytes to a new image file, or an image into a bdev nothing has open yet; not part of the
		 * configuration dump, since an image is data, not state */
		if (!decode(params, {{"name", Json::Str, false, &a}, {"path", Json::Str, false, &b}})) return bad;
		oimgpu_image_info info;
		int rc = method == "save_bdev_image" ? oimgpu_bdev_image_save(a->raw.c_str(), b->raw.c_str(), &info)
						     : oimgpu_bdev_image_load(a->raw.c_str(), b->raw.c_str(), &info);
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		return result(id, "{\"name\":" + jstr(a->raw) + ",\"path\":" + jstr(b->raw) +
				  ",\"block_size\":" + std::to_string(info.block_size) + ",\"num_blocks\":" + std::to_string(info.num_blocks) +
				  ",\"uuid\":" + jstr(info.uuid) + ",\"extents\":" + std::to_string(info.nextents) +
				  ",\"data_bytes\":" + std::to_string(info.data_bytes) + ",\"file_bytes\":" + std::to_string(info.file_bytes) + "}");
	}
	if (method == "enable_bdev_image_tracking") {
		/* keep the fingerprints a delta is taken against; like the images, not part of the configuration dump */
		if (!decode(params, {{"name", Json::Str, false, &a}, {"enable", Json::Bool, true, &b}})) return bad;
		int rc = oimgpu_bdev_image_track(a->raw.c_str(), b ? b->b : 1);
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		return result(id, "true");
	}
	if (method == "save_bdev_image_delta" || method == "apply_bdev_image_delta") {
		/* the granules a tracked bdev changed since its last save or load, to a new delta file; or a delta into a bdev
		 * nothing has open yet whose content is the delta's parent */
		if (!decode(params, {{"name", Json::Str, false, &a}, {"path", Json::Str, false, &b}})) return bad;
		oimgpu_image_delta_info info;
		int rc = method == "save_bdev_image_delta" ? oimgpu_bdev_image_save_delta(a->raw.c_str(), b->raw.c_str(), &info)
							   : oimgpu_bdev_image_apply_delta(a->raw.c_str(), b->raw.c_str(), &info);
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		auto hex = [](const uint64_t d[2]) {
			char s[33];
			snprintf(s, sizeof(s), "%016llx%016llx", (unsigned long long)d[0], (unsigned long long)d[1]);
			return jstr(s);
		};
		return result(id, "{\"name\":" + jstr(a->raw) + ",\"path\":" + jstr(b->raw) +
				  ",\"block_size\":" + std::to_string(info.block_size) + ",\"num_blocks\":" + std::to_string(info.num_blocks) +
				  ",\"uuid\":" + jstr(info.uuid) + ",\"extents\":" + std::to_string(info.nextents) +
				  ",\"data_bytes\":" + std::to_string(info.data_bytes) + ",\"zero_bytes\":" + std::to_string(info.zero_bytes) +
				  ",\"file_bytes\":" + std::to_string(info.file_bytes) + ",\"parent_digest\":" + hex(info.parent_digest) +
				  ",\"digest\":" + hex(info.digest) + "}");
	}
	if (method == "delete_bdev") {
		if (!decode(params, {{"name", Json::Str, false, &a}})) return bad;
		/* the SCSI targets built on the bdev go with it (spdk_bdev_unregister -> hot-remove, lun.c:213-260); connected
		 * guests are told like for remove_vhost_scsi_target (TRANSPORT_RESET / REMOVED, vhost_scsi.c:236-289) */
		std::vector<std::pair<std::string, int>> gone;
		if (g_serve_vhost_user) {
			int n = oimgpu_vhost_ctrlr_list(nullptr, 0);
			std::vector<oimgpu_ctrlr_info> v(n > 0 ? n : 1);
			n = oimgpu_vhost_ctrlr_list(v.data(), n);
			for (int i = 0; i < n; i++) {
				for (uint32_t t = 0; t < v[i].ntargets; t++) {
					if (a->raw == v[i].targets[t].bdev_name) gone.push_back({v[i].ctrlr, v[i].targets[t].scsi_dev_num});
				}
			}
		}
		if (oimgpu_bdev_delete(a->raw.c_str()) != 0) return bad;
		for (auto &g : gone) vhost_user::notify_target(g.first, g.second, false);
		return result(id, "true");
	}
	if (method == "construct_vhost_scsi_controller") {
		if (!decode(params, {{"ctrlr", Json::Str, false, &a}, {"cpumask", Json::Str, true, &b}}))
			return error(id, E_INVALID_PARAMS, strerr(EINVAL));
		int rc = oimgpu_vhost_scsi_ctrlr_create(a->raw.c_str(), b ? b->raw.c_str() : nullptr);
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		/* spdk_vhost_dev_register: the controller's vhost-user socket appears at <socket dir><name> (vhost.c:715-760) */
		oimgpu_ctrlr_info info;
		if (g_serve_vhost_user && oimgpu_vhost_ctrlr_get(a->raw.c_str(), &info) == 0) {
			rc = vhost_user::listen_ctrlr(info.ctrlr, info.socket);
			if (rc < 0) {
				oimgpu_vhost_ctrlr_remove(a->raw.c_str());
				return error(id, E_INVALID_PARAMS, strerr(rc));
			}
		}
		return result(id, "true");
	}
	if (method == "add_vhost_scsi_lun") {
		int32_t num = 0;
		if (!decode(params, {{"ctrlr", Json::Str, false, &a}, {"scsi_target_num", Json::Num, false, &b}, {"bdev_name", Json::Str, false, &c}}) ||
		    !to_i32(b, &num)) return error(id, E_INVALID_PARAMS, strerr(EINVAL));
		int rc = oimgpu_vhost_scsi_add_lun(a->raw.c_str(), num, c->raw.c_str());
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		oimgpu_ctrlr_info info;
		if (g_serve_vhost_user && oimgpu_vhost_ctrlr_get(a->raw.c_str(), &info) == 0) vhost_user::notify_target(info.ctrlr, rc, true);
		return result(id, std::to_string(rc));
	}
	if (method == "remove_vhost_scsi_target") {
		uint64_t num = 0;
		if (!decode(params, {{"ctrlr", Json::Str, false, &a}, {"scsi_target_num", Json::Num, false, &b}}) ||
		    !to_u64(b, &num) || num > UINT32_MAX) return error(id, E_INVALID_PARAMS, strerr(EINVAL));
		int rc = oimgpu_vhost_scsi_remove_target(a->raw.c_str(), num > INT32_MAX ? INT32_MAX : (int)num);
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		oimgpu_ctrlr_info info;
		if (g_serve_vhost_user && oimgpu_vhost_ctrlr_get(a->raw.c_str(), &info) == 0) vhost_user::notify_target(info.ctrlr, (int)num, false);
		return result(id, "true");
	}
	if (method == "remove_vhost_controller") {
		if (!decode(params, {{"ctrlr", Json::Str, false, &a}})) return error(id, E_INVALID_PARAMS, strerr(EINVAL));
		oimgpu_ctrlr_info info;
		const bool known = oimgpu_vhost_ctrlr_get(a->raw.c_str(), &info) == 0;
		/* spdk_vhost_dev_unregister: "Controller %s has still valid connection" -> -EBUSY (S/lib/vhost/vhost.c:783-788) */
		if (g_serve_vhost_user && known && vhost_user::active_sessions(info.ctrlr) > 0) return error(id, E_INVALID_PARAMS, strerr(EBUSY));
		int rc = oimgpu_vhost_ctrlr_remove(a->raw.c_str());
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		if (g_serve_vhost_user && known) vhost_user::close_ctrlr(info.ctrlr);
		return result(id, "true");
	}
	if (method == "set_vhost_controller_coalescing") {
		/* S/lib/vhost/vhost_rpc.c:493-544 */
		uint64_t delay = 0, thr = 0;
		if (!decode(params, {{"ctrlr", Json::Str, false, &a}, {"delay_base_us", Json::Num, false, &b}, {"iops_threshold", Json::Num, false, &c}}) ||
		    !to_u64(b, &delay) || !to_u64(c, &thr) || delay > UINT32_MAX || thr > UINT32_MAX)
			return error(id, E_INVALID_PARAMS, strerr(EINVAL));
		int rc = oimgpu_vhost_ctrlr_set_coalescing(a->raw.c_str(), (uint32_t)delay, (uint32_t)thr);
		if (rc < 0) return error(id, E_INVALID_PARAMS, strerr(rc));
		return result(id, "true");
	}
	if (method == "get_subsystems") {
		/* S/lib/event/rpc/subsystem_rpc.c:40-78, the subsystems this daemon has */
		return result(id, "[{\"subsystem\":\"copy\",\"depends_on\":[]},{\"subsystem\":\"bdev\",\"depends_on\":[\"copy\"]},"
				  "{\"subsystem\":\"scsi\",\"depends_on\":[\"bdev\"]},{\"subsystem\":\"vhost\",\"depends_on\":[\"scsi\"]}]");
	}
	if (method == "get_subsystem_config") {
		if (!decode(params, {{"name", Json::Str, false, &a}})) return error(id, E_INVALID_PARAMS, "Invalid arguments");
		if (a->raw == "copy" || a->raw == "scsi") return result(id, "[]");
		long n = oimgpu_config_json(a->raw.c_str(), nullptr, 0);
		if (n < 0) return error(id, E_INVALID_PARAMS, "Subsystem '" + a->raw + "' not found");
		std::string buf((size_t)n + 1, '\0');
		oimgpu_config_json(a->raw.c_str(), &buf[0], buf.size());
		buf.resize((size_t)n);
		return result(id, buf);
	}
	if (method == "get_vhost_controllers") {
		if (params && !decode(params, {{"name", Json::Str, true, &a}})) return error(id, E_INTERNAL, strerr(EINVAL));
		std::string out = "[";
		if (a) {
			oimgpu_ctrlr_info info;
			if (oimgpu_vhost_ctrlr_get(a->raw.c_str(), &info) != 0) return error(id, E_INTERNAL, strerr(ENODEV));
			out += ctrlr_json(info);
		} else {
			int n = oimgpu_vhost_ctrlr_list(nullptr, 0);
			std::vector<oimgpu_ctrlr_info> v(n > 0 ? n : 1);
			n = oimgpu_vhost_ctrlr_list(v.data(), n);
			for (int i = 0; i < n; i++) out += (i ? "," : "") + ctrlr_json(v[i]);
		}
		return result(id, out + "]");
	}
	/* NBD export needs the kernel nbd module + root and moves data through the CPU; OIM's "local" mode
	 * (pkg/oim-csi-driver/local.go:119-206) is the only user.  The names are served so the shims get a
	 * well-formed answer (S/lib/nbd/nbd_rpc.c:62-311 shapes); start reports ENOTSUP. */
	if (method == "get_nbd_disks") {
		if (params && !decode(params, {{"nbd_device", Json::Str, true, &a}})) return bad;
		std::string out = "[";
		bool first = true;
		for (auto &n : g_nbd) {
			if (a && n->dev != a->raw) continue;
			out += std::string(first ? "" : ",") + "{\"nbd_device\":" + jstr(n->dev) + ",\"bdev_name\":" + jstr(n->bdev) + "}";
			first = false;
		}
		if (a && first) return bad;
		return result(id, out + "]");
	}
	if (method == "start_nbd_disk") {
		if (!decode(params, {{"bdev_name", Json::Str, false, &a}, {"nbd_device", Json::Str, false, &b}})) return bad;
		for (auto &n : g_nbd) if (n->dev == b->raw) return bad;	/* already exported */
		if (nbd_start(a->raw, b->raw) != 0) return bad;		/* nbd_rpc.c:63-70: whatever went wrong */
		return result(id, jstr(b->raw));
	}
	if (method == "stop_nbd_disk") {
		if (!decode(params, {{"nbd_device", Json::Str, false, &a}})) return bad;
		for (size_t i = 0; i < g_nbd.size(); i++) {
			if (g_nbd[i]->dev != a->raw) continue;
			nbd_stop(*g_nbd[i]);
			g_nbd.erase(g_nbd.begin() + i);
			return result(id, "true");
		}
		return bad;	/* no such NBD device */
	}
	return error(id, E_METHOD_NOT_FOUND, "Method not found");
}

/* parse_single_request (jsonrpc_server.c:62-101) */
static Reply handle(const Json &v)
{
	if (v.type != Json::Obj) return error(nullptr, E_INVALID_REQUEST, "Invalid request");
	const Json *ver = nullptr, *method = nullptr, *params = nullptr, *id = nullptr;
	bool ok = true;
	int seen[4] = {0, 0, 0, 0};
	for (auto &kv : v.obj) {
		if (kv.first == "jsonrpc") { ver = &kv.second; if (seen[0]++) ok = false; }
		else if (kv.first == "method") { method = &kv.second; if (seen[1]++) ok = false; }
		else if (kv.first == "params") { params = &kv.second; if (seen[2]++) ok = false; }
		else if (kv.first == "id") { id = &kv.second; if (seen[3]++) ok = false; }
		else ok = false;
	}
	const Json *rid = (id && (id->type == Json::Str || id->type == Json::Num || id->type == Json::Null)) ? id : nullptr;
	if (!ok) return error(nullptr, E_INVALID_REQUEST, "Invalid request");
	if (ver && (ver->type != Json::Str || ver->raw != "2.0")) return error(nullptr, E_INVALID_REQUEST, "Invalid request");
	if (!method || method->type != Json::Str) return error(nullptr, E_INVALID_REQUEST, "Invalid request");
	if (id && !rid) return error(nullptr, E_INVALID_REQUEST, "Invalid request");
	if (params && params->type != Json::Arr && params->type != Json::Obj) return error(rid, E_INVALID_REQUEST, "Invalid request");
	return dispatch(method->raw, params, rid);
}

/* ---- socket server -------------------------------------------------------------------------------- */

struct Conn { int fd; std::string in, out; bool closing = false; };
static volatile sig_atomic_t g_stop = 0;
static void on_signal(int) { g_stop = 1; }

static void usage(const char *argv0)
{
	fprintf(stderr,
		"usage: %s [-S vhost-socket-dir] [-r rpc-socket] [-f pidfile] [-m coremask] [-s MB] [-R]\n"
		"       [--gpus 0,1,...] [--rbd-size BYTES] [--poller] [--no-vhost-user] [--control-only]\n"
		"  -S -r -f -m -s -R   as SPDK's vhost app (S/app/vhost/vhost.c:43-48); -s and -R are accepted and ignored\n"
		"  --gpus LIST         CUDA devices to serve bdevs from (default: the current device)\n"
		"  --rbd-size BYTES    size of a construct_rbd_bdev volume (emulated in HBM; default 8 GiB)\n"
		"  --poller            one resident GPU poller per vhost-user session instead of a launch per kick\n"
		"  --no-vhost-user     JSON-RPC only: do not listen on <vhost-socket-dir>/<controller>\n"
		"  --control-only      no CUDA at all: bookkeeping and wire protocols only (tests)\n"
		"  environment: OIM_VU_DEBUG=1 logs session start/stop; SIGUSR2 prints the transport threads' backtraces\n",
		argv0);
}

int main(int argc, char **argv)
{
	std::string rpc_sock = "/var/tmp/spdk.sock", sock_dir, pidfile, coremask;
	std::vector<int> gpus;
	bool control_only = false;
	vhost_user::Config vu_cfg;
	for (int i = 1; i < argc; i++) {
		std::string a = argv[i];
		auto next = [&]() -> const char * { return i + 1 < argc ? argv[++i] : ""; };
		if (a == "-S") sock_dir = next();
		else if (a == "-r") rpc_sock = next();
		else if (a == "-f") pidfile = next();
		else if (a == "-m") coremask = next();
		else if (a == "-s") next();
		else if (a == "-R") {}
		else if (a == "--control-only") control_only = true;	/* protocol tests without a GPU: no data path */
		else if (a == "--poller") vu_cfg.poller = true;		/* a resident GPU poller per vhost-user session */
		else if (a == "--no-vhost-user") g_serve_vhost_user = false;
		else if (a == "--no-spread") vu_cfg.spread = false;	/* several GPUs: keep a session on the GPU of its first target */
		else if (a == "--rbd-size") g_rbd_default_size = strtoull(next(), nullptr, 0);
		else if (a == "--gpus") {
			std::string l = next();
			for (size_t p = 0; p < l.size();) {
				size_t q = l.find(',', p);
				gpus.push_back(atoi(l.substr(p, q - p).c_str()));
				if (q == std::string::npos) break;
				p = q + 1;
			}
		} else { usage(argv[0]); return 2; }
	}
	vu_cfg.control_only = control_only;
	vhost_user::configure(vu_cfg);
	int rc = control_only ? oimgpu_init_control_only() : oimgpu_init(gpus.empty() ? nullptr : gpus.data(), (int)gpus.size());
	if (rc != 0) {
		fprintf(stderr, "oim-gpu-vhost: oimgpu_init failed: %s\n", strerror(-rc));
		return 1;
	}
	if (coremask.compare(0, 2, "0x") == 0) coremask = coremask.substr(2);
	if (oimgpu_set_socket_dir(sock_dir.c_str(), coremask.c_str()) != 0) { fprintf(stderr, "bad -m\n"); return 2; }

	int lfd = socket(AF_UNIX, SOCK_STREAM, 0);
	sockaddr_un sa{};
	sa.sun_family = AF_UNIX;
	/* bind under a temporary name and rename once listening: whoever waits for the socket file to appear
	 * (test/pkg/spdk/spdk.go:121-133, start-stop.make:17) can connect the moment it does */
	const std::string rpc_tmp = rpc_sock + ".starting";
	snprintf(sa.sun_path, sizeof(sa.sun_path), "%s", rpc_tmp.c_str());
	unlink(rpc_tmp.c_str());
	if (rpc_tmp.size() >= sizeof(sa.sun_path) || bind(lfd, (sockaddr *)&sa, sizeof(sa)) != 0 || listen(lfd, 64) != 0 ||
	    rename(rpc_tmp.c_str(), rpc_sock.c_str()) != 0) {
		fprintf(stderr, "oim-gpu-vhost: cannot listen on %s: %s\n", rpc_sock.c_str(), strerror(errno));
		return 1;
	}
	if (!pidfile.empty()) {
		FILE *f = fopen(pidfile.c_str(), "w");
		if (f) { fprintf(f, "%d\n", getpid()); fclose(f); }
	}
	signal(SIGINT, on_signal);
	signal(SIGTERM, on_signal);
	signal(SIGPIPE, SIG_IGN);
	fprintf(stderr, "oim-gpu-vhost: %s, %d GPU(s), RPC socket %s\n", oimgpu_version_string(), oimgpu_device_count(), rpc_sock.c_str());

	std::vector<Conn> conns;
	while (!g_stop) {
		std::vector<pollfd> pfds;
		pfds.push_back({lfd, POLLIN, 0});
		for (auto &c : conns) pfds.push_back({c.fd, (short)(POLLIN | (c.out.empty() ? 0 : POLLOUT)), 0});
		if (poll(pfds.data(), pfds.size(), 200) < 0) continue;
		if (pfds[0].revents & POLLIN) {
			int fd = accept(lfd, nullptr, nullptr);
			if (fd >= 0) { fcntl(fd, F_SETFL, O_NONBLOCK); conns.push_back({fd, "", ""}); }
		}
		for (size_t i = 0; i < conns.size() && i + 1 < pfds.size(); i++) {
			Conn &c = conns[i];
			if (pfds[i + 1].revents & (POLLIN | POLLHUP)) {
				char buf[65536];
				ssize_t n = read(c.fd, buf, sizeof(buf));
				if (n > 0) c.in.append(buf, n);
				else if (n == 0 || (errno != EAGAIN && errno != EINTR)) c.closing = true;
				/* the peer is gone for good (not a half-close): whatever is still queued has nowhere to go */
				if ((pfds[i + 1].revents & (POLLHUP | POLLERR)) && n <= 0) { c.closing = true; c.out.clear(); }
			}
			/* requests are processed in order per connection; one JSON value at a time */
			while (!c.in.empty()) {
				Parser ps{c.in.data(), c.in.data() + c.in.size()};
				Json v;
				const char *start = ps.p;
				ps.ws();
				if (ps.p == ps.end) { c.in.clear(); break; }
				bool ok = ps.value(v);
				if (!ok && ps.incomplete) {
					/* wait for the rest - but not for ever: the reference's receive buffer is 32 KiB
					 * (SPDK_JSONRPC_RECV_BUF_SIZE, jsonrpc_internal.h:43); a value that does not fit is a
					 * parse error there, and the connection goes */
					if (c.in.size() > 32 * 1024) { c.in.clear(); c.closing = true; }
					break;
				}
				if (!ok) {
					/* "Can't recover from parse error (no guaranteed resync point in streaming JSON)":
					 * the reference queues a -32700 reply but closes the connection before it is
					 * flushed (jsonrpc_server.c:151-159 returns -1), so the peer just sees EOF */
					c.in.clear();
					c.closing = true;
					break;
				}
				c.in.erase(0, ps.p - start);
				Reply r = handle(v);
				if (r.has) c.out += r.body;
			}
			if (!c.out.empty()) {
				ssize_t n = write(c.fd, c.out.data(), c.out.size());
				if (n > 0) c.out.erase(0, n);
				else if (n < 0 && errno != EAGAIN && errno != EINTR) { c.closing = true; c.out.clear(); }	/* EPIPE: drop the reply */
			}
		}
		for (size_t i = 0; i < conns.size();) {
			if (conns[i].closing && conns[i].out.empty()) { close(conns[i].fd); conns.erase(conns.begin() + i); }
			else i++;
		}
	}
	for (auto &c : conns) close(c.fd);
	for (auto &n : g_nbd) nbd_stop(*n);
	g_nbd.clear();
	vhost_user::shutdown();
	close(lfd);
	unlink(rpc_sock.c_str());
	if (!pidfile.empty()) unlink(pidfile.c_str());
	oimgpu_fini();
	return 0;
}
