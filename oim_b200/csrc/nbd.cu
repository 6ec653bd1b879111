/*
 * nbd.cu - NBD export (S/lib/nbd/nbd.c): OIM's local mode without a VM.
 */
#include <sys/socket.h>
#include <unistd.h>

#include "host_state.h"

static bool read_full(int fd, void *buf, size_t n)
{
	size_t got = 0;
	while (got < n) {
		ssize_t r = read(fd, (char *)buf + got, n - got);
		if (r < 0 && errno == EINTR) continue;
		if (r <= 0) return false;
		got += (size_t)r;
	}
	return true;
}

static bool write_full(int fd, const void *buf, size_t n)
{
	size_t put = 0;
	while (put < n) {
		ssize_t r = send(fd, (const char *)buf + put, n - put, MSG_NOSIGNAL);
		if (r < 0 && errno == EINTR) continue;
		if (r <= 0) return false;
		put += (size_t)r;
	}
	return true;
}

/* Serve the kernel's NBD transmission protocol on `sock_fd` (the daemon's end of the socketpair whose
 * other end went to /dev/nbdX with NBD_SET_SOCK) until the peer disconnects: struct nbd_request in,
 * struct nbd_reply (+ payload for reads) out, as spdk_nbd_poll does (nbd.c:560-806).  The store stays
 * in HBM; payload crosses a pinned bounce buffer with the copy engine - this is a CPU-socket path by
 * nature (the reference moves every byte through the same socket), not a hot path.
 * Returns 0 on an orderly end (NBD_CMD_DISC or EOF), -EINVAL on a bad request magic, -errno otherwise. */
extern "C" int oimgpu_nbd_serve(const char *bdev_name, int sock_fd)
{
	std::vector<Replica> reps;
	uint64_t size = 0;
	uint32_t bs = 0;
	std::string name = bdev_name ? bdev_name : "";
	{
		std::lock_guard<std::mutex> lk(g.mu);
		if (!g.inited || g.control_only) return -ENODEV;
		Bdev *b = find_bdev_locked(name.c_str());
		if (!b) return -ENODEV;
		reps = b->replicas;
		size = b->num_blocks * (uint64_t)b->block_size;
		bs = b->block_size;
		open_bdev_locked(*b);	/* a use like a session's */
		b->nbd_exports++;	/* and refuses a mirror check: this loop cannot be paused */
	}
	int rc = 0;
	cudaStream_t st = nullptr;
	Buf<uint8_t, Mem::Pinned> bounce;
	cudaSetDevice(reps[0].device);
	if (cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking) != cudaSuccess) rc = -EIO;
	auto book = [&](int op, uint64_t bytes) {	/* get_bdevs_iostat counts these like any other bdev I/O */
		std::lock_guard<std::mutex> lk(g.mu);
		Bdev *b = find_bdev_locked(name.c_str());
		if (!b) return;
		b->retired[op] += 1;
		b->retired[4 + op] += bytes;
	};
	while (rc == 0) {
		uint8_t req[28];	/* struct nbd_request: magic, type, handle[8], from, len - big endian */
		if (!read_full(sock_fd, req, sizeof(req))) break;
		auto be32 = [](const uint8_t *p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; };
		if (be32(req) != 0x25609513u) { rc = -EINVAL; break; }
		const uint32_t type = be32(req + 4), len = be32(req + 24);
		uint64_t from = 0;
		for (int k = 0; k < 8; k++) from = from << 8 | req[16 + k];
		const uint32_t payload = (type == 0 || type == 1) ? len : 0;	/* only READ / WRITE carry one */
		if (payload > bounce.size()) {
			std::lock_guard<std::mutex> lk(g.mu);
			const size_t cap = ((size_t)payload + (1u << 20) - 1) & ~(size_t)((1u << 20) - 1);
			if (bounce.grow(reps[0].device, cap, ParkedPollers(bounce.waits_for())) != cudaSuccess) { rc = -ENOMEM; break; }
		}
		if (type == 1 && payload && !read_full(sock_fd, bounce.get(), payload)) break;
		if (type == 2) break;	/* NBD_CMD_DISC: nothing outstanding here, close */
		/* spdk_bdev_bytes_to_blocks + spdk_bdev_io_valid_blocks (bdev.c:2474-2509): whole blocks, inside the device */
		const bool range_ok = from % bs == 0 && len % bs == 0 && from <= size && len <= size - from;
		bool ok = false;
		cudaError_t e = cudaSuccess;
		switch (type) {
		case 0:		/* NBD_CMD_READ */
			ok = range_ok;
			if (ok && payload) e = cudaMemcpyAsync(bounce.get(), reps[0].store + from, payload, cudaMemcpyDeviceToHost, st);
			break;
		case 1:		/* NBD_CMD_WRITE */
			ok = range_ok;
			for (size_t r = 0; ok && payload && r < reps.size() && e == cudaSuccess; r++)
				e = cudaMemcpyAsync(reps[r].store + from, bounce.get(), payload, cudaMemcpyHostToDevice, st);
			break;
		case 3:		/* NBD_CMD_FLUSH: the whole device, a no-op for RAM */
			ok = true;
			break;
		case 4:		/* NBD_CMD_TRIM -> spdk_bdev_unmap: zero fill; "Can't unmap 0 bytes" (bdev.c:2796-2799) */
			ok = range_ok && len != 0;
			for (size_t r = 0; ok && len && r < reps.size() && e == cudaSuccess; r++) e = cudaMemsetAsync(reps[r].store + from, 0, len, st);
			break;
		default:	/* unknown command: EIO (nbd.c:527-540) */
			break;
		}
		if (e == cudaSuccess) e = cudaStreamSynchronize(st);
		if (e != cudaSuccess) { (void)cudaGetLastError(); ok = false; }
		if (ok && (type == 0 || type == 1 || type == 4)) book(type == 0 ? 0 : type == 1 ? 1 : 2, len);
		uint8_t resp[16] = {0x67, 0x44, 0x66, 0x98, 0, 0, 0, (uint8_t)(ok ? 0 : EIO)};	/* struct nbd_reply */
		memcpy(resp + 8, req + 8, 8);
		if (!write_full(sock_fd, resp, sizeof(resp))) break;
		if (type == 0 && ok && payload && !write_full(sock_fd, bounce.get(), payload)) break;
	}
	{
		std::lock_guard<std::mutex> lk(g.mu);
		bounce.reset(ParkedPollers(bounce.waits_for()));
		close_bdev_locked(name);
		Bdev *b = find_bdev_locked(name.c_str());
		if (b && b->nbd_exports > 0) b->nbd_exports--;
	}
	if (st) cudaStreamDestroy(st);
	return rc;
}

