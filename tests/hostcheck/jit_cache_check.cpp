/*
 * jit_cache_check: drives the on-disk kernel cache (dragnet_b200/csrc/
 * jit_cache.h) without a GPU, for tests/test_jit_cache_host.py.  Built with
 * g++ -Werror together with jit_cache.cpp.  One command per line on stdin,
 * one line of output per command:
 *
 *   put DIR KEY CUBIN BOUND NAME   store; CUBIN = @path (a file's bytes) or a
 *                                  byte count (a pattern made from KEY);
 *                                  NAME = - for the key's own file name
 *   get DIR KEY NAME [OUT]         look up (OUT: write the cubin found there)
 *   forge DIR KEY CUBIN NAME FMT   write an entry in format version FMT
 *   fork N DIR KEY CUBIN BOUND     N processes put KEY at once
 *   age DIR NAME SECONDS           set a file's mtime SECONDS into the past
 *   name KEY                       the key's file name
 *   buildid PATH                   the build id of a library file
 *   stats                          the process's counters
 */
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <sys/stat.h>
#include <sys/wait.h>
#include <time.h>
#include <unistd.h>

#include <fstream>
#include <iostream>
#include <sstream>
#include <string>

#include "jit_cache.h"

using namespace dng;

static std::string cubin_of(const std::string &spec, const std::string &key)
{
	if (!spec.empty() && spec[0] == '@') {
		std::ifstream f(spec.substr(1), std::ios::binary);
		std::stringstream ss;
		ss << f.rdbuf();
		return ss.str();
	}
	std::string c(strtoull(spec.c_str(), nullptr, 10), '\0');
	for (size_t i = 0; i < c.size(); i++)
		c[i] = (char)(key[i % key.size()] + i / key.size());
	return c;
}

static std::string name_of(const std::string &name, const std::string &key)
{
	return name == "-" ? jit_cache_name(key) : name;
}

int main()
{
	std::string line;
	while (std::getline(std::cin, line)) {
		std::istringstream in(line);
		std::string cmd, dir, key, spec, name, out;
		in >> cmd;
		if (cmd == "put") {
			unsigned long long bound;
			in >> dir >> key >> spec >> bound >> name;
			const bool ok = jit_cache_put(dir, name_of(name, key), key,
			    cubin_of(spec, key), bound);
			printf("ok=%d\n", ok ? 1 : 0);
		} else if (cmd == "get") {
			in >> dir >> key >> name >> out;
			std::string c;
			const bool hit = jit_cache_get(dir, name_of(name, key), key,
			    c);
			if (hit && !out.empty())
				std::ofstream(out, std::ios::binary) << c;
			printf("hit=%d bytes=%zu same=%d\n", hit ? 1 : 0, c.size(),
			    hit && c == cubin_of(std::to_string(c.size()), key) ?
			    1 : 0);
		} else if (cmd == "forge") {
			unsigned fmt;
			in >> dir >> key >> spec >> name >> fmt;
			std::ofstream(dir + "/" + name_of(name, key),
			    std::ios::binary) << jit_cache_entry(key,
			    cubin_of(spec, key), fmt);
			printf("ok=1\n");
		} else if (cmd == "fork") {
			int n;
			unsigned long long bound;
			in >> n >> dir >> key >> spec >> bound;
			const std::string c = cubin_of(spec, key);
			for (int i = 0; i < n; i++)
				if (fork() == 0)
					_exit(jit_cache_put(dir, jit_cache_name(key),
					    key, c, bound) ? 0 : 1);
			int failed = 0, st;
			while (wait(&st) > 0)
				failed += !WIFEXITED(st) || WEXITSTATUS(st) != 0;
			printf("failed=%d\n", failed);
		} else if (cmd == "age") {
			long secs;
			in >> dir >> name >> secs;
			struct timespec ts[2];
			clock_gettime(CLOCK_REALTIME, &ts[0]);
			ts[0].tv_sec -= secs;
			ts[1] = ts[0];
			const std::string p = dir + "/" + name;
			printf("ok=%d\n", utimensat(AT_FDCWD, p.c_str(), ts, 0) == 0);
		} else if (cmd == "name") {
			in >> key;
			printf("name=%s\n", jit_cache_name(key).c_str());
		} else if (cmd == "buildid") {
			in >> dir;
			const std::string id = jit_cache_build_id(dir.c_str());
			printf("id=%s\n", id.empty() ? "-" : id.c_str());
		} else if (cmd == "stats") {
			const JitCacheStats s = jit_cache_stats();
			printf("hits=%llu misses=%llu writes=%llu evictions=%llu "
			    "errors=%llu\n", (unsigned long long)s.hits,
			    (unsigned long long)s.misses,
			    (unsigned long long)s.writes,
			    (unsigned long long)s.evictions,
			    (unsigned long long)s.errors);
		} else {
			fprintf(stderr, "unknown command: %s\n", line.c_str());
			return 2;
		}
		fflush(stdout);
	}
	return 0;
}
