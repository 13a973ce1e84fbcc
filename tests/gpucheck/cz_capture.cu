/*
 * cz_capture: the library's compressed-input object (compressed.o, built
 * from dragnet_b200/csrc/compressed.cu) run with stubs in place of the six
 * functions it takes from api.cu, keeping every byte it feeds the scan
 * (TEST ONLY; tests/test_gpu_decode_bytes.py).
 *
 *   cz_capture MANIFEST OUTDIR
 *
 * MANIFEST is text, one scan after another:
 *
 *   scan NAME SM_COUNT POISON CAPACITY
 *   gz PATH | bz PATH        (one line per file, fed in order)
 *   end
 *
 * SM_COUNT 0 is the device's; POISON is the byte every buffer the decoders
 * allocate is filled with; CAPACITY bounds the bytes captured.  Per scan,
 * OUTDIR/<index>.bin gets the fed bytes back to back, and OUTDIR/results
 * one JSON line: the feeds' return codes, the scan's error, each feed's
 * length and alignment, the gzip, split and bzip2 stats, and the frees made
 * while the scan's stream still had work queued.
 *
 * Nothing here synchronises the scan's stream on the decoders' behalf: a fed
 * buffer is copied out by a cudaMemcpyAsync queued on that stream, so it is
 * read when the scan's kernels would read it, and a buffer overwritten before
 * then shows up as wrong bytes.  Frees are deferred to the end of a scan, as
 * cudaFree would synchronise the device.
 */
#include <cuda_runtime.h>
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <string>
#include <utility>
#include <vector>

#include "scan.h"

static dng_scan *cur;		/* the scan being run */
static int poison;
static uint8_t *capture;	/* pinned, CAPACITY bytes */
static size_t capture_cap, captured;
static bool overflow;
static std::vector<std::pair<uint64_t, int>> feeds;	/* length, aligned */
static std::vector<std::pair<void *, bool>> deferred;	/* pointer, device */
static uint64_t busy_frees;

cudaError_t dng_cached_alloc(int device, void **p, size_t n)
{
	cudaError_t e;
	if (device < 0) {
		e = cudaMallocHost(p, n);
		if (e == cudaSuccess)
			memset(*p, poison, n);
	} else {
		e = cudaMalloc(p, n);
		if (e == cudaSuccess)
			e = cudaMemsetAsync(*p, poison, n, cur->stream);
	}
	return e;
}

void dng_cached_free(void *p)
{
	if (!p)
		return;
	cudaPointerAttributes a;
	const bool dev = cudaPointerGetAttributes(&a, p) == cudaSuccess &&
	    a.type == cudaMemoryTypeDevice;
	if (cudaStreamQuery(cur->stream) == cudaErrorNotReady)
		busy_frees++;
	deferred.push_back({ p, dev });
}

cudaEvent_t get_event(dng_scan *)
{
	cudaEvent_t e;
	cudaEventCreate(&e);
	return e;
}

/* as api.cu's: not sticky, the scan goes on */
int refuse_multi(dng_scan *s, const char *what)
{
	if (!s->err_code)
		s->err = std::string(what) + " on a scan over several devices";
	return DNG_EINVAL;
}

/* dng_scan_feed_device's contract, then the bytes copied out on the stream */
int feed_device(dng_scan *s, const void *devbuf, size_t len)
{
	if (s->err_code)
		return s->err_code;
	if (s->finished)
		return s->fail(DNG_EINVAL, "scan already finished");
	const int aligned = !((uintptr_t)devbuf & 15);
	feeds.push_back({ len, aligned });
	if (!aligned)
		return s->fail(DNG_EINVAL, "device buffer must be 16-byte "
		    "aligned");
	if (!len)
		return 0;
	if (captured + len > capture_cap) {
		overflow = true;
		return 0;
	}
	s->bytes_fed += len;
	CK(s, cudaMemcpyAsync(capture + captured, devbuf, len,
	    cudaMemcpyDeviceToHost, s->stream));
	captured += len;
	return 0;
}

int read_to_device(dng_scan *s, const char *path, size_t size, dng::u8 *dst)
{
	std::vector<uint8_t> buf(size);
	int fd = open(path, O_RDONLY);
	if (fd < 0)
		return s->fail(DNG_EIO, std::string("open ") + path);
	size_t got = 0;
	while (got < size) {
		ssize_t r = pread(fd, buf.data() + got, size - got, got);
		if (r <= 0)
			break;
		got += (size_t)r;
	}
	close(fd);
	if (got != size)
		return s->fail(DNG_EIO, std::string(path) + ": short read");
	/* on the scan's stream, as the library's reader copies: after the
	 * poison memset of the batch buffer, before the decoders read it (a
	 * copy from pageable memory returns once `buf` is staged) */
	CK(s, cudaMemcpyAsync(dst, buf.data(), size, cudaMemcpyHostToDevice,
	    s->stream));
	return 0;
}

static std::string quote(const std::string &v)
{
	std::string o = "\"";
	for (unsigned char c : v) {
		if (c == '"' || c == '\\') {
			o += '\\';
			o += (char)c;
		} else if (c < 0x20) {
			char b[8];
			snprintf(b, sizeof b, "\\u%04x", c);
			o += b;
		} else {
			o += (char)c;
		}
	}
	return o + "\"";
}

template <size_t N> static std::string list(const uint64_t (&v)[N])
{
	std::string o = "[";
	for (size_t i = 0; i < N; i++)
		o += (i ? "," : "") + std::to_string(v[i]);
	return o + "]";
}

struct Scan {
	std::string name;
	int sm = 0, poison = 0;
	size_t cap = 0;
	std::vector<std::pair<bool, std::string>> files;	/* bzip2, path */
};

int main(int argc, char **argv)
{
	if (argc != 3) {
		fprintf(stderr, "usage: cz_capture MANIFEST OUTDIR\n");
		return 2;
	}
	FILE *m = fopen(argv[1], "r");
	if (!m) {
		perror(argv[1]);
		return 2;
	}
	std::vector<Scan> scans;
	char line[8192];
	while (fgets(line, sizeof line, m)) {
		line[strcspn(line, "\n")] = 0;
		if (!strncmp(line, "scan ", 5)) {
			Scan sc;
			char name[4096];
			if (sscanf(line + 5, "%4095s %d %i %zu", name, &sc.sm,
			    &sc.poison, &sc.cap) != 4)
				return 2;
			sc.name = name;
			scans.push_back(sc);
		} else if (!strncmp(line, "gz ", 3) || !strncmp(line, "bz ", 3)) {
			if (scans.empty())
				return 2;
			scans.back().files.push_back({ line[0] == 'b', line + 3 });
		} else if (strcmp(line, "end") && line[0]) {
			fprintf(stderr, "bad manifest line: %s\n", line);
			return 2;
		}
	}
	fclose(m);
	size_t cap = 1;
	for (const Scan &sc : scans)
		cap = std::max(cap, sc.cap);
	if (cudaMallocHost(&capture, cap) != cudaSuccess) {
		fprintf(stderr, "no pinned capture buffer of %zu bytes\n", cap);
		return 3;
	}
	cudaDeviceProp prop;
	cudaGetDeviceProperties(&prop, 0);
	const std::string out = argv[2];
	FILE *res = fopen((out + "/results").c_str(), "w");
	if (!res)
		return 2;
	for (size_t k = 0; k < scans.size(); k++) {
		const Scan &sc = scans[k];
		printf("scan %zu %s\n", k, sc.name.c_str());
		fflush(stdout);
		poison = sc.poison;
		capture_cap = sc.cap;
		captured = 0;
		overflow = false;
		feeds.clear();
		busy_frees = 0;
		dng_scan *s = new dng_scan();
		cur = s;
		s->device = 0;
		s->sm_count = sc.sm ? sc.sm : prop.multiProcessorCount;
		cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking);
		std::string rcs = "[";
		for (size_t i = 0; i < sc.files.size(); i++) {
			const char *p = sc.files[i].second.c_str();
			const int rc = sc.files[i].first ?
			    dng_scan_feed_bzip2(s, p) : dng_scan_feed_gzip(s, p);
			rcs += (i ? "," : "") + std::to_string(rc);
		}
		rcs += "]";
		const int flush = cz_flush(s);
		const cudaError_t se = cudaStreamSynchronize(s->stream);
		if (se != cudaSuccess)
			s->cuda(se, "cudaStreamSynchronize");
		s->finished = true;
		uint64_t gz[5], sp[5], bz[7];
		double ms;
		dng_scan_gzip_stats(s, &gz[0], &gz[1], &gz[2], &gz[3], &gz[4], &ms);
		dng_scan_gzip_split_stats(s, &sp[0], &sp[1], &sp[2], &sp[3],
		    &sp[4]);
		dng_scan_bzip2_stats(s, &bz[0], &bz[1], &bz[2], &bz[3], &bz[4],
		    &bz[5], &bz[6], &ms);
		std::string fl = "[";
		for (size_t i = 0; i < feeds.size(); i++)
			fl += std::string(i ? "," : "") + "[" +
			    std::to_string(feeds[i].first) + "," +
			    std::to_string(feeds[i].second) + "]";
		fl += "]";
		cz_free(s->cz);
		s->cz = nullptr;
		cudaStreamSynchronize(s->stream);
		for (auto &d : deferred)
			if (d.second)
				cudaFree(d.first);
			else
				cudaFreeHost(d.first);
		deferred.clear();
		for (cudaEvent_t e : s->ev_pool)
			cudaEventDestroy(e);
		cudaStreamDestroy(s->stream);
		fprintf(res, "{\"name\":%s,\"rcs\":%s,\"flush\":%d,\"err_code\":%d,"
		    "\"err\":%s,\"feeds\":%s,\"captured\":%zu,\"overflow\":%d,"
		    "\"gzip\":%s,\"split\":%s,\"bzip2\":%s,\"busy_frees\":%llu}\n",
		    quote(sc.name).c_str(), rcs.c_str(), flush, s->err_code,
		    quote(s->err).c_str(), fl.c_str(), captured, (int)overflow,
		    list(gz).c_str(), list(sp).c_str(), list(bz).c_str(),
		    (unsigned long long)busy_frees);
		fflush(res);
		FILE *b = fopen((out + "/" + std::to_string(k) + ".bin").c_str(),
		    "wb");
		if (!b || (captured && fwrite(capture, 1, captured, b) != captured))
			return 2;
		fclose(b);
		const bool sticky = s->err_code == DNG_ECUDA;
		delete s;
		if (sticky)
			return 4;	/* a sticky error: no later scan is worth it */
	}
	fclose(res);
	cudaFreeHost(capture);
	return 0;
}
