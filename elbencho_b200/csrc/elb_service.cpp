/*
 * Distributed mode implementation (see elb_service.h).
 */
#include <arpa/inet.h>
#include <errno.h>
#include <fcntl.h>
#include <netdb.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <poll.h>
#include <pwd.h>
#include <signal.h>
#include <string.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <sys/time.h>
#include <sys/types.h>
#include <unistd.h>

#include <algorithm>
#include <fstream>
#include <iostream>
#include <random>
#include <sstream>
#include <thread>

#include "elb_service.h"
#include "elb_worker.h"

#define ELB_BENCHPATH_DELIMITER ",\n\r@" /* source/ProgArgs.cpp:42 */
#define ELB_SVC_UPDATE_INTERVAL_MS 500   /* source/ProgArgs.cpp:969 svcUpdateIntervalMS */
#define ELB_HTTP_MAX_REQUEST_BYTES (64 * 1024 * 1024)

namespace elb
{

/* ==============================================================================================
 * JsonTree
 * ============================================================================================ */

const JsonTree* JsonTree::find(const std::string& path) const
{
	const JsonTree* node = this;
	size_t start = 0;

	while(start <= path.size() )
	{
		size_t dotPos = path.find('.', start);
		const std::string key = path.substr(start,
			(dotPos == std::string::npos) ? std::string::npos : (dotPos - start) );

		const JsonTree* next = NULL;

		for(const std::pair<std::string, JsonTree>& child : node->children)
			if(child.first == key)
			{
				next = &child.second;
				break;
			}

		if(!next)
			return NULL;

		node = next;

		if(dotPos == std::string::npos)
			break;

		start = dotPos + 1;
	}

	return node;
}

JsonTree* JsonTree::findOrCreate(const std::string& path, bool alwaysAppendLeaf)
{
	JsonTree* node = this;
	size_t start = 0;

	for( ; ; )
	{
		size_t dotPos = path.find('.', start);
		const bool isLeaf = (dotPos == std::string::npos);
		const std::string key = path.substr(start, isLeaf ? std::string::npos : (dotPos - start) );

		JsonTree* next = NULL;

		if(!(isLeaf && alwaysAppendLeaf) )
			for(std::pair<std::string, JsonTree>& child : node->children)
				if(child.first == key)
				{
					next = &child.second;
					break;
				}

		if(!next)
		{
			node->children.emplace_back(key, JsonTree() );
			next = &node->children.back().second;
		}

		node = next;

		if(isLeaf)
			return node;

		start = dotPos + 1;
	}
}

void JsonTree::put(const std::string& path, const std::string& newValue)
{
	findOrCreate(path, false)->value = newValue;
}

void JsonTree::add(const std::string& path, const std::string& newValue)
{
	findOrCreate(path, true)->value = newValue;
}

std::string JsonTree::getStr(const std::string& path) const
{
	const JsonTree* node = find(path);

	if(!node)
		throw ProgError("No such node (" + path + ")"); // (boost ptree_bad_path text)

	return node->value;
}

std::string JsonTree::getStr(const std::string& path, const std::string& defaultValue) const
{
	const JsonTree* node = find(path);
	return node ? node->value : defaultValue;
}

uint64_t JsonTree::getU64(const std::string& path) const
{
	const std::string raw = getStr(path);
	char* endPtr = NULL;
	const uint64_t parsed = strtoull(raw.c_str(), &endPtr, 10);

	if(raw.empty() || (endPtr && *endPtr) )
		throw ProgError("conversion of data to type failed (" + path + "=" + raw + ")");

	return parsed;
}

uint64_t JsonTree::getU64(const std::string& path, uint64_t defaultValue) const
{
	return has(path) ? getU64(path) : defaultValue;
}

bool JsonTree::getBool(const std::string& path) const
{
	const std::string raw = getStr(path);

	if( (raw == "true") || (raw == "1") )
		return true;

	if( (raw == "false") || (raw == "0") )
		return false;

	throw ProgError("conversion of data to type failed (" + path + "=" + raw + ")");
}

bool JsonTree::getBool(const std::string& path, bool defaultValue) const
{
	return has(path) ? getBool(path) : defaultValue;
}

static void jsonEscapeInto(std::string& out, const std::string& raw)
{
	for(unsigned char c : raw)
	{
		switch(c)
		{
			case '"': out += "\\\""; break;
			case '\\': out += "\\\\"; break;
			case '/': out += "\\/"; break;
			case '\b': out += "\\b"; break;
			case '\f': out += "\\f"; break;
			case '\n': out += "\\n"; break;
			case '\r': out += "\\r"; break;
			case '\t': out += "\\t"; break;
			default:
				if(c < 0x20)
				{
					char buf[8];
					snprintf(buf, sizeof(buf), "\\u%04X", c);
					out += buf;
				}
				else
					out += (char)c;
		}
	}
}

void JsonTree::write(std::string& out, bool pretty, int indent) const
{
	if(children.empty() )
	{
		out += "\"";
		jsonEscapeInto(out, value);
		out += "\"";
		return;
	}

	out += "{";

	for(size_t i = 0; i < children.size(); i++)
	{
		if(pretty)
			out += "\n" + std::string( (indent + 1) * 4, ' ');

		out += "\"";
		jsonEscapeInto(out, children[i].first);
		out += pretty ? "\": " : "\":";

		children[i].second.write(out, pretty, indent + 1);

		if(i < (children.size() - 1) )
			out += ",";
	}

	if(pretty)
		out += "\n" + std::string(indent * 4, ' ');

	out += "}";
}

std::string JsonTree::toJSON(bool pretty) const
{
	std::string out;

	if(children.empty() && value.empty() )
		out = "{}";
	else
		write(out, pretty, 0);

	if(pretty)
		out += "\n";

	return out;
}

/* recursive descent parser: objects, arrays (elements get empty keys like ptree), strings,
 * numbers/true/false/null (kept as their text) */
class JsonParser
{
	public:
		explicit JsonParser(const std::string& text) : text(text) {}

		JsonTree parseDocument()
		{
			JsonTree tree = parseValue();
			skipWhitespace();

			if(pos != text.size() )
				fail("garbage after data");

			return tree;
		}

	private:
		const std::string& text;
		size_t pos{0};

		[[noreturn]] void fail(const std::string& what)
		{
			throw ProgError("JSON parse error at offset " + std::to_string(pos) + ": " + what);
		}

		void skipWhitespace()
		{
			while( (pos < text.size() ) && isspace( (unsigned char)text[pos] ) )
				pos++;
		}

		char peek()
		{
			skipWhitespace();

			if(pos >= text.size() )
				fail("unexpected end of data");

			return text[pos];
		}

		std::string parseString()
		{
			if(peek() != '"')
				fail("expected string");

			pos++;

			std::string out;

			while(pos < text.size() )
			{
				char c = text[pos++];

				if(c == '"')
					return out;

				if(c != '\\')
				{
					out += c;
					continue;
				}

				if(pos >= text.size() )
					break;

				char esc = text[pos++];

				switch(esc)
				{
					case 'n': out += '\n'; break;
					case 't': out += '\t'; break;
					case 'r': out += '\r'; break;
					case 'b': out += '\b'; break;
					case 'f': out += '\f'; break;
					case 'u':
					{
						if( (pos + 4) > text.size() )
							fail("bad unicode escape");

						unsigned codePoint = (unsigned)strtoul(text.substr(pos, 4).c_str(), NULL, 16);
						pos += 4;

						if(codePoint < 0x80)
							out += (char)codePoint;
						else
						if(codePoint < 0x800)
						{
							out += (char)(0xC0 | (codePoint >> 6) );
							out += (char)(0x80 | (codePoint & 0x3F) );
						}
						else
						{
							out += (char)(0xE0 | (codePoint >> 12) );
							out += (char)(0x80 | ( (codePoint >> 6) & 0x3F) );
							out += (char)(0x80 | (codePoint & 0x3F) );
						}
					} break;
					default: out += esc; break; // \" \\ \/
				}
			}

			fail("unterminated string");
		}

		JsonTree parseValue()
		{
			char c = peek();

			if(c == '{')
			{
				pos++;
				JsonTree tree;

				if(peek() == '}')
				{
					pos++;
					return tree;
				}

				for( ; ; )
				{
					std::string key = parseString();

					if(peek() != ':')
						fail("expected ':'");

					pos++;

					JsonTree child = parseValue();
					appendChild(tree, key, child);

					char next = peek();
					pos++;

					if(next == '}')
						return tree;

					if(next != ',')
						fail("expected ',' or '}'");
				}
			}

			if(c == '[')
			{
				pos++;
				JsonTree tree;

				if(peek() == ']')
				{
					pos++;
					return tree;
				}

				for( ; ; )
				{
					JsonTree child = parseValue();
					appendChild(tree, "", child);

					char next = peek();
					pos++;

					if(next == ']')
						return tree;

					if(next != ',')
						fail("expected ',' or ']'");
				}
			}

			if(c == '"')
				return JsonTree(parseString() );

			// bare literal: number, true, false, null
			size_t start = pos;

			while( (pos < text.size() ) && (isalnum( (unsigned char)text[pos] ) ||
				(text[pos] == '-') || (text[pos] == '+') || (text[pos] == '.') ) )
				pos++;

			if(start == pos)
				fail("unexpected character");

			std::string literal = text.substr(start, pos - start);

			return JsonTree( (literal == "null") ? "" : literal);
		}

		static void appendChild(JsonTree& parent, const std::string& key, const JsonTree& child);
};

/* (friend-free: rebuild through the public add/put interface would lose subtrees, so JsonTree
 * exposes its children vector read-only and the parser builds via this helper) */
void JsonParser::appendChild(JsonTree& parent, const std::string& key, const JsonTree& child)
{
	const_cast<JsonTree::ChildVec&>(parent.getChildren() ).emplace_back(key, child);
}

JsonTree JsonTree::parse(const std::string& text)
{
	JsonParser parser(text);
	return parser.parseDocument();
}

/* ==============================================================================================
 * HTTP
 * ============================================================================================ */

std::string urlEncode(const std::string& raw)
{
	std::string out;
	char buf[4];

	for(unsigned char c : raw)
	{
		if(isalnum(c) || (c == '-') || (c == '_') || (c == '.') || (c == '~') )
			out += (char)c;
		else
		{
			snprintf(buf, sizeof(buf), "%%%02X", c);
			out += buf;
		}
	}

	return out;
}

static std::string urlDecode(const std::string& raw)
{
	std::string out;

	for(size_t i = 0; i < raw.size(); i++)
	{
		if( (raw[i] == '%') && ( (i + 2) < raw.size() ) )
		{
			out += (char)strtoul(raw.substr(i + 1, 2).c_str(), NULL, 16);
			i += 2;
		}
		else
		if(raw[i] == '+')
			out += ' ';
		else
			out += raw[i];
	}

	return out;
}

static void parseQuery(const std::string& queryStr, std::map<std::string, std::string>& out)
{
	std::stringstream queryStream(queryStr);
	std::string item;

	while(std::getline(queryStream, item, '&') )
	{
		if(item.empty() )
			continue;

		const size_t eqPos = item.find('=');

		if(eqPos == std::string::npos)
			out[urlDecode(item)] = "";
		else
			out[urlDecode(item.substr(0, eqPos) )] = urlDecode(item.substr(eqPos + 1) );
	}
}

static bool sendAll(int sock, const std::string& data)
{
	size_t numSent = 0;

	while(numSent < data.size() )
	{
		ssize_t sendRes = send(sock, data.data() + numSent, data.size() - numSent, MSG_NOSIGNAL);

		if(sendRes <= 0)
		{
			if( (sendRes < 0) && (errno == EINTR) )
				continue;

			return false;
		}

		numSent += sendRes;
	}

	return true;
}

static const char* httpStatusText(int statusCode)
{
	switch(statusCode)
	{
		case 200: return "OK";
		case 400: return "Bad Request";
		case 404: return "Not Found";
		default: return "Error";
	}
}

/* parsed view of a (possibly still incomplete) HTTP message in a receive buffer */
struct HttpMessageView
{
	bool complete{false};
	bool invalid{false};   // e.g. a Content-Length beyond what this server accepts
	size_t totalLen{0};
	size_t neededLen{0};   // bytes the buffer must hold before the message can be complete
	std::string startLine;
	std::map<std::string, std::string> headers; // lower-case names
	std::string body;
};

static HttpMessageView parseHttpMessage(const std::string& buffer, bool bodyUntilClose,
	bool connectionClosed)
{
	HttpMessageView view;

	const size_t headerEnd = buffer.find("\r\n\r\n");
	if(headerEnd == std::string::npos)
		return view;

	std::stringstream headerStream(buffer.substr(0, headerEnd) );
	std::string line;

	std::getline(headerStream, line);
	if(!line.empty() && (line.back() == '\r') )
		line.pop_back();
	view.startLine = line;

	while(std::getline(headerStream, line) )
	{
		if(!line.empty() && (line.back() == '\r') )
			line.pop_back();

		const size_t colonPos = line.find(':');
		if(colonPos == std::string::npos)
			continue;

		std::string name = line.substr(0, colonPos);
		std::transform(name.begin(), name.end(), name.begin(), ::tolower);

		size_t valueStart = colonPos + 1;
		while( (valueStart < line.size() ) && (line[valueStart] == ' ') )
			valueStart++;

		view.headers[name] = line.substr(valueStart);
	}

	const size_t bodyStart = headerEnd + 4;

	if(view.headers.count("content-length") )
	{
		const unsigned long long contentLen =
			strtoull(view.headers["content-length"].c_str(), NULL, 10);

		if(contentLen > ELB_HTTP_MAX_REQUEST_BYTES)
		{ // (checked before any arithmetic with it)
			view.invalid = true;
			return view;
		}

		view.neededLen = bodyStart + (size_t)contentLen;

		if(buffer.size() < view.neededLen)
			return view;

		view.body = buffer.substr(bodyStart, contentLen);
		view.totalLen = bodyStart + contentLen;
		view.complete = true;
	}
	else
	if(bodyUntilClose)
	{ // response without length: body ends when the peer closes
		if(!connectionClosed)
			return view;

		view.body = buffer.substr(bodyStart);
		view.totalLen = buffer.size();
		view.complete = true;
	}
	else
	{ // request without body
		view.totalLen = bodyStart;
		view.complete = true;
	}

	return view;
}

HttpResponse httpRequest(const std::string& host, unsigned short port, const std::string& method,
	const std::string& pathAndQuery, const std::string& body, int timeoutSecs)
{
	struct addrinfo hints;
	struct addrinfo* addrList = NULL;
	memset(&hints, 0, sizeof(hints) );
	hints.ai_family = AF_UNSPEC;
	hints.ai_socktype = SOCK_STREAM;

	int addrRes = getaddrinfo(host.c_str(), std::to_string(port).c_str(), &hints, &addrList);
	if(addrRes)
		throw ProgError("Unable to resolve host: " + host + "; Error: " + gai_strerror(addrRes) );

	int sock = -1;
	std::string connectErr;

	for(struct addrinfo* addr = addrList; addr; addr = addr->ai_next)
	{
		sock = socket(addr->ai_family, addr->ai_socktype, addr->ai_protocol);
		if(sock == -1)
			continue;

		struct timeval timeout = {timeoutSecs, 0};
		setsockopt(sock, SOL_SOCKET, SO_RCVTIMEO, &timeout, sizeof(timeout) );
		setsockopt(sock, SOL_SOCKET, SO_SNDTIMEO, &timeout, sizeof(timeout) );

		if(connect(sock, addr->ai_addr, addr->ai_addrlen) == 0)
			break;

		connectErr = strerror(errno);
		close(sock);
		sock = -1;
	}

	freeaddrinfo(addrList);

	if(sock == -1)
		throw ProgError("Unable to connect to service. Host: " + host + ":" +
			std::to_string(port) + "; SysErr: " + connectErr);

	int enable = 1;
	setsockopt(sock, IPPROTO_TCP, TCP_NODELAY, &enable, sizeof(enable) );

	std::string request = method + " " + pathAndQuery + " HTTP/1.1\r\n"
		"Host: " + host + ":" + std::to_string(port) + "\r\n"
		"Connection: close\r\n"
		"Content-Length: " + std::to_string(body.size() ) + "\r\n\r\n" + body;

	if(!sendAll(sock, request) )
	{
		close(sock);
		throw ProgError("Sending request to service failed. Host: " + host);
	}

	std::string buffer;
	char chunk[65536];
	bool closed = false;
	HttpMessageView view;

	while(!view.complete)
	{
		ssize_t recvRes = recv(sock, chunk, sizeof(chunk), 0);

		if(recvRes < 0)
		{
			if(errno == EINTR)
				continue;

			close(sock);
			throw ProgError("Receiving response from service failed. Host: " + host + "; SysErr: " +
				strerror(errno) );
		}

		if(recvRes == 0)
			closed = true;
		else
			buffer.append(chunk, recvRes);

		view = parseHttpMessage(buffer, true, closed);

		if(closed && !view.complete)
		{
			close(sock);
			throw ProgError("Service closed connection before sending a complete response. "
				"Host: " + host);
		}
	}

	close(sock);

	HttpResponse response;
	response.body = view.body;

	// "HTTP/1.1 200 OK"
	const size_t spacePos = view.startLine.find(' ');
	response.statusCode = (spacePos == std::string::npos) ?
		0 : atoi(view.startLine.c_str() + spacePos + 1);

	return response;
}

/* ==============================================================================================
 * Service side (HTTPServiceSWS.cpp)
 * ============================================================================================ */

class Service
{
	public:
		explicit Service(ProgArgs& progArgs) :
			progArgs(progArgs), svcPasswordHash(progArgs.svcPasswordHash) {}

		int run();

	private:
		ProgArgs& progArgs;
		std::unique_ptr<Manager> manager;
		ProgArgs::ABIConfig abiConfig;
		std::vector<std::string> benchPaths;
		std::string benchPathStr;
		std::string currentBenchID;
		int currentPhase{ELB_PHASE_IDLE};
		std::string errHistory;
		bool quitRequested{false};
		CPUUtil liveCpuUtil;
		bool isRWMixConfig{false};
		Clock::time_point phaseStartT;

		HttpResponse handle(const HttpRequest& request);
		HttpResponse handlePreparePhase(const HttpRequest& request);
		HttpResponse handlePrepareFile(const HttpRequest& request);
		void checkAuthorization(const HttpRequest& request) const;
		std::string svcPasswordHash; // of this service's own --svcpwfile (kept over prepare phases)
		std::string uploadBasePath() const;
		HttpResponse handleStartPhase(const HttpRequest& request);
		HttpResponse handleStatus();
		HttpResponse handleBenchResult();
		HttpResponse handleInterruptPhase(const HttpRequest& request);
		void resetManager();
		void collectErrHistory();
		void putCommonStats(JsonTree& tree, bool isFinal,
			const elb_live_snapshot* liveSnapshot = NULL);
};

void Service::resetManager()
{
	manager.reset(); // interrupts + joins the workers, closes paths (HTTPServiceSWS.cpp:432-437)
}

void Service::collectErrHistory()
{
	if(!manager)
		return;

	for(const std::unique_ptr<Worker>& worker : manager->workers)
	{
		const std::string workerErr = worker->getLastError();

		if(!workerErr.empty() && (errHistory.find(workerErr) == std::string::npos) )
			errHistory += "ERROR: " + workerErr + "\n";
	}
}

static void histogramToTree(const elb_histogram& histo, const std::string& prefix, JsonTree& tree)
{ // LatencyHistogram::getAsPropertyTreeForService (LatencyHistogram.cpp:68-79)
	tree.put(prefix + "LatNumValues", histo.numStoredValues);
	tree.put(prefix + "LatMicroSecTotal", histo.numMicroSecTotal);
	tree.put(prefix + "LatMinMicroSec", histo.minMicroSecLat);
	tree.put(prefix + "LatMaxMicroSec", histo.maxMicroSecLat);

	for(size_t i = 0; i < ELB_LATHISTO_NUMBUCKETS; i++)
		tree.add(prefix + "LatHistoList.item", histo.buckets[i] );
}

static void histogramFromTree(const JsonTree& tree, const std::string& prefix, elb_histogram& histo)
{ // LatencyHistogram::setFromPropertyTreeForService (LatencyHistogram.cpp:84-97)
	histogramReset(histo);
	histo.numStoredValues = tree.getU64(prefix + "LatNumValues");
	histo.numMicroSecTotal = tree.getU64(prefix + "LatMicroSecTotal");
	histo.minMicroSecLat = tree.getU64(prefix + "LatMinMicroSec");
	histo.maxMicroSecLat = tree.getU64(prefix + "LatMaxMicroSec");

	const JsonTree* listNode = tree.find(prefix + "LatHistoList");
	size_t bucketIndex = 0;

	if(listNode)
		for(const std::pair<std::string, JsonTree>& item : listNode->getChildren() )
		{
			if(bucketIndex >= ELB_LATHISTO_NUMBUCKETS)
				break;

			histo.buckets[bucketIndex++] = strtoull(item.second.getValue().c_str(), NULL, 10);
		}
}

/* common part of /status and /benchresult (Statistics.cpp:1350-1405, 2728-2804) */
void Service::putCommonStats(JsonTree& tree, bool isFinal, const elb_live_snapshot* liveSnapshot)
{
	elb_liveops liveOps[2] = {};
	size_t numWorkersDone = 0, numWorkersDoneWithError = 0;
	bool stoneWallTriggered = false;

	if(manager)
	{
		if(liveSnapshot)
		{
			liveOps[0] = liveSnapshot->ops;
			liveOps[1] = liveSnapshot->opsReadMix;
		}
		else
			for(const std::unique_ptr<Worker>& worker : manager->workers)
			{
				liveOpsAdd(liveOps[0], worker->getLiveOps() );
				liveOpsAdd(liveOps[1], worker->getLiveOpsReadMix() );
			}

		std::unique_lock<std::mutex> lock(manager->shared.mutex);
		numWorkersDoneWithError = manager->shared.numWorkersDoneWithError;
		/* (the reference counts workers with error separately from numWorkersDone,
		   WorkersSharedData.cpp:36-44) */
		numWorkersDone = manager->shared.numWorkersDone - numWorkersDoneWithError;
		stoneWallTriggered = !manager->workers.empty() &&
			manager->workers[0]->getStoneWallTriggered();
	}

	tree.put("BenchID", currentBenchID);
	tree.put("PhaseName", stats::phaseName(currentPhase, progArgs) );
	tree.put("PhaseCode", (uint64_t)currentPhase);
	tree.put("NumWorkersDone", numWorkersDone);
	tree.put("NumWorkersDoneWithError", numWorkersDoneWithError);

	if(!isFinal)
		tree.putBool("TriggerStoneWall", stoneWallTriggered);

	tree.put("NumEntriesDone", liveOps[0].numEntriesDone);
	tree.put("NumBytesDone", liveOps[0].numBytesDone);
	tree.put("NumIOPSDone", liveOps[0].numIOPSDone);

	if(isRWMixConfig && (currentPhase == ELB_PHASE_CREATEFILES) )
	{
		tree.put("NumEntriesDoneRWMixRead", liveOps[1].numEntriesDone);
		tree.put("NumBytesDoneRWMixRead", liveOps[1].numBytesDone);
		tree.put("NumIOPSDoneRWMixRead", liveOps[1].numIOPSDone);
	}
}

HttpResponse Service::handleStatus()
{
	JsonTree tree;
	HttpResponse response;

	/* workers on several GPUs: per-GPU partial sums reduced over NVLink by NCCL
	   (LiveStatsReducer); final results always come from the exact per-worker values */
	elb_live_snapshot liveSnapshot;
	const bool useLiveReduce = manager && (manager->getNumGPUs() >= 2);

	if(useLiveReduce)
		manager->getLiveSnapshot(liveSnapshot);

	/* phase time limit: the master polls /status every few hundred ms, so this is where the
	   service notices the expiry and asks its workers to finish (friendly interruption, the
	   results stay; WorkerManager::checkPhaseTimeLimit, WorkerManager.cpp:109-128) */
	if(manager && progArgs.timeLimitSecs && (currentPhase != ELB_PHASE_IDLE) &&
		( (uint64_t)std::chrono::duration_cast<std::chrono::seconds>(
			Clock::now() - phaseStartT).count() >= progArgs.timeLimitSecs) )
	{
		std::unique_lock<std::mutex> lock(manager->shared.mutex);

		for(Worker* worker : manager->shared.workers)
			worker->interruptExecution();
	}

	putCommonStats(tree, false, useLiveReduce ? &liveSnapshot : NULL);

	liveCpuUtil.update();
	tree.put("CPUUtil", liveCpuUtil.getCPUUtilPercent() );
	tree.put("ElapsedSecs", (uint64_t)std::chrono::duration_cast<std::chrono::seconds>(
		Clock::now() - phaseStartT).count() );

	elb_livelat liveLat = {};
	if(useLiveReduce)
		liveLat = liveSnapshot.lat;
	else
	if(manager)
		for(const std::unique_ptr<Worker>& worker : manager->workers)
			worker->getAndResetLiveLatency(liveLat);

	tree.put("NumIOLatUSec", liveLat.numAvgIOLatValues);
	tree.put("SumIOLatUSec", liveLat.avgIOLatMicroSecsSum);
	tree.put("NumEntLatUSec", liveLat.numAvgEntriesLatValues);
	tree.put("SumEntLatUSec", liveLat.avgEntriesLatMicroSecsSum);

	if(isRWMixConfig && (currentPhase == ELB_PHASE_CREATEFILES) )
	{
		tree.put("NumIOLatUSecRWMixRead", (uint64_t)0);
		tree.put("SumIOLatUSecRWMixRead", (uint64_t)0);
		tree.put("NumEntLatUSecRWMixRead", (uint64_t)0);
		tree.put("SumEntLatUSecRWMixRead", (uint64_t)0);
	}

	collectErrHistory();
	tree.put("ErrorHistory", errHistory);

	response.body = tree.toJSON();
	return response;
}

HttpResponse Service::handleBenchResult()
{
	JsonTree tree;
	HttpResponse response;

	if(!manager)
	{
		response.statusCode = 400;
		response.body = "Benchmark results requested, but no phase was prepared.";
		return response;
	}

	putCommonStats(tree, true);

	elb_phase_results res;
	manager->getPhaseResults(res);

	tree.put("CPUUtilStoneWall", res.cpuUtilStoneWallPercent);
	tree.put("CPUUtil", res.cpuUtilPercent);

	bool triggerStonewall = false;

	for(const std::unique_ptr<Worker>& worker : manager->workers)
	{
		if(!worker->getWorkerGotPhaseWork() )
			continue;

		triggerStonewall = true;

		if(worker->getElapsedUSec() )
			tree.add("ElapsedUSecList.item", worker->getElapsedUSec() );
	}

	tree.putBool("TriggerStoneWall", triggerStonewall);

	histogramToTree(res.iopsLatHisto, "IOPS_", tree);
	histogramToTree(res.entriesLatHisto, "Entries_", tree);

	if(isRWMixConfig && (currentPhase == ELB_PHASE_CREATEFILES) )
	{
		histogramToTree(res.iopsLatHistoReadMix, "IOPSRWMixRead_", tree);
		histogramToTree(res.entriesLatHistoReadMix, "EntriesRWMixRead_", tree);
	}

	collectErrHistory();
	tree.put("ErrorHistory", errHistory);

	// show results when running in foreground (HTTPServiceSWS.cpp:241)
	std::vector<uint64_t> elapsedUSecVec;
	for(const std::unique_ptr<Worker>& worker : manager->workers)
		if(worker->getElapsedUSec() )
			elapsedUSecVec.push_back(worker->getElapsedUSec() );

	if(!elapsedUSecVec.empty() )
	{
		stats::printPhaseResults(progArgs, currentPhase, res, elapsedUSecVec, std::cout);
		std::cout << std::endl;
	}

	response.body = tree.toJSON();
	return response;
}

/* ProgArgs::setFromPropertyTreeForService (ProgArgs.cpp:3562-3680), supported subset; unknown
 * keys are ignored, missing keys take the defaults */
/* authorization hash of the master vs ours (HTTPServiceSWS.cpp:287-296, 400-409) */
void Service::checkAuthorization(const HttpRequest& request) const
{
	if(!request.query.count("PwHash") )
		throw ProgError("Missing parameter: PwHash");

	if(request.query.at("PwHash") != svcPasswordHash)
		throw ProgError("Invalid authorization code.");
}

/* SERVICE_UPLOAD_BASEPATH (ProgArgs.h:228-230): /var/tmp/<exe>_<user>_p<port> */
std::string Service::uploadBasePath() const
{
	const char* userName = getenv("USER");
	struct passwd* passwdEntry = getpwuid(geteuid() );

	if(passwdEntry && passwdEntry->pw_name)
		userName = passwdEntry->pw_name;

	return std::string("/var/tmp/elbencho-b200_") + (userName ? userName : "unknown") + "_p" +
		std::to_string(progArgs.servicePort);
}

/* receive input files for the following prepare phase, i.e. the custom tree file
 * (HTTPServiceSWS.cpp:262-350) */
HttpResponse Service::handlePrepareFile(const HttpRequest& request)
{
	HttpResponse response;

	try
	{
		if(!request.query.count("ProtocolVersion") )
			throw ProgError("Missing parameter: ProtocolVersion");

		const std::string masterProtoVer = request.query.at("ProtocolVersion");
		if(masterProtoVer != ELB_HTTP_PROTOCOLVERSION)
			throw ProgError("Protocol version mismatch. "
				"Service version: " ELB_HTTP_PROTOCOLVERSION "; "
				"Received master version: " + masterProtoVer);

		checkAuthorization(request);

		if(!request.query.count("FileName") )
			throw ProgError("Missing parameter: FileName");

		// (only the last path component: no "../" or subdirs in the given filename)
		std::string filename = request.query.at("FileName");
		const size_t slashPos = filename.find_last_of('/');

		if(slashPos != std::string::npos)
			filename = filename.substr(slashPos + 1);

		if(filename.empty() || (filename == ".") || (filename == "..") )
			throw ProgError("Invalid file name: " + request.query.at("FileName") );

		const std::string basePath = uploadBasePath();
		const std::string path = basePath + "/" + filename;

		std::cout << "Receiving tree file from master..." << std::endl;

		if( (mkdir(basePath.c_str(), 0700) == -1) && (errno != EEXIST) )
			throw ProgError("Failed to create service tmp dir: " + basePath);

		/* the directory name is predictable: only use it if it is a real directory of this user,
		   and never write through a symlink somebody else placed there */
		struct stat dirStat;

		if( (lstat(basePath.c_str(), &dirStat) == -1) || !S_ISDIR(dirStat.st_mode) ||
			(dirStat.st_uid != geteuid() ) )
			throw ProgError("Service tmp dir is not a directory owned by this user: " + basePath);

		const int uploadFD = open(path.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_NOFOLLOW, 0600);

		if(uploadFD == -1)
			throw ProgError("Opening upload file failed: " + path + "; SysErr: " + strerror(errno) );

		size_t numWritten = 0;

		while(numWritten < request.body.size() )
		{
			const ssize_t writeRes = write(uploadFD, request.body.data() + numWritten,
				request.body.size() - numWritten);

			if(writeRes <= 0)
			{
				close(uploadFD);
				throw ProgError("Saving upload file failed: " + path);
			}

			numWritten += writeRes;
		}

		if(close(uploadFD) == -1)
			throw ProgError("Saving upload file failed: " + path);
	}
	catch(std::exception& e)
	{
		response.statusCode = 400;
		response.body = std::string("File preparation phase error: ") + e.what() + "\n";
		std::cerr << "ERROR: " << response.body;
	}

	return response;
}

HttpResponse Service::handlePreparePhase(const HttpRequest& request)
{
	HttpResponse response;

	try
	{
		if(!request.query.count("ProtocolVersion") )
			throw ProgError("Missing parameter: ProtocolVersion");

		const std::string masterProtoVer = request.query.at("ProtocolVersion");
		if(masterProtoVer != ELB_HTTP_PROTOCOLVERSION)
			throw ProgError("Protocol version mismatch. "
				"Service version: " ELB_HTTP_PROTOCOLVERSION "; "
				"Received master version: " + masterProtoVer);

		checkAuthorization(request);

		time_t currentTime = time(NULL);
		struct tm localTimeInfo;
		localtime_r(&currentTime, &localTimeInfo);
		char dateBuf[64];
		strftime(dateBuf, sizeof(dateBuf), "%FT%T%z", &localTimeInfo);

		std::cout << "Preparing new benchmark phase... (ISO DATE: " << dateBuf << ")" << std::endl;

		JsonTree recvTree = JsonTree::parse(request.body);

		resetManager();
		errHistory.clear();

		ProgArgs& args = progArgs;

		args.benchLabel = recvTree.getStr("label", "");
		benchPathStr = recvTree.getStr("path");
		args.blockSize = recvTree.getU64("block");
		args.blockVariancePercent = recvTree.getU64("blockvarpct", 0);
		args.doDirectVerify = recvTree.getBool("verifydirect", false);
		args.doDirSharing = recvTree.getBool("dirsharing", false);
		args.doPreallocFile = recvTree.getBool("preallocfile", false);
		args.doReadInline = recvTree.getBool("readinline", false);
		args.doReverseSeqOffsets = recvTree.getBool("backward", false);
		args.doTruncate = recvTree.getBool("trunc", false);
		args.doTruncToSize = recvTree.getBool("trunctosize", false);
		args.fileSize = recvTree.getU64("size");
		args.gpuIDsStr = recvTree.getStr("gpuids", "");
		args.ignoreDelErrors = recvTree.getBool("nodelerr", false);
		args.integrityCheckSalt = recvTree.getU64("verify", 0);
		args.fadviseFlags = recvTree.getU64("fadv", 0);
		args.flockType = recvTree.getU64("flock", 0);
		args.doStatInline = recvTree.getBool("statinline", false);
		args.noDirectIOCheck = recvTree.getBool("nodiocheck", false);
		args.doInfiniteIOLoop = recvTree.getBool("infloop", false);
		args.timeLimitSecs = recvTree.getU64("b200_timelimit", 0);
		args.limitReadBps = recvTree.getU64("limitread", 0);
		args.limitWriteBps = recvTree.getU64("limitwrite", 0);
		args.ioDepth = recvTree.getU64("iodepth", 1);
		args.numDirs = recvTree.getU64("dirs", 1);
		args.numFiles = recvTree.getU64("files", 1);
		args.numRWMixReadThreads = recvTree.getU64("rwmixthr", 0);
		args.hasUserSetRWMixReadThreads = (args.numRWMixReadThreads != 0);
		args.rwMixThreadsReadPercent = recvTree.getU64("rwmixthrpct", 0);
		args.numThreads = recvTree.getU64("threads", 1);
		args.randOffsetAlgo = recvTree.getStr("randalgo", "");
		args.randomAmount = recvTree.getU64("randamount", 0);
		args.rankOffset = recvTree.getU64("rankoffset", 0);
		args.runCreateDirsPhase = recvTree.getBool("mkdirs", false);
		args.runCreateFilesPhase = recvTree.getBool("write", false);
		args.runDeleteDirsPhase = recvTree.getBool("deldirs", false);
		args.runDeleteFilesPhase = recvTree.getBool("delfiles", false);
		args.runDropCachesPhase = recvTree.getBool("dropcache", false);
		args.runReadPhase = recvTree.getBool("read", false);
		args.runStatFilesPhase = recvTree.getBool("stat", false);
		args.runSyncPhase = recvTree.getBool("sync", false);
		args.rwMixReadPercent = recvTree.getU64("rwmixpct", 0);
		args.hasUserSetRWMixPercent = (args.rwMixReadPercent != 0);
		args.useCuFile = recvTree.getBool("cufile", false);
		args.useDirectIO = recvTree.getBool("direct", false);
		args.useGDSBufReg = recvTree.getBool("gdsbufreg", false);
		args.useRandomOffsets = recvTree.getBool("rand", false);
		args.useRandomUnaligned = recvTree.getBool("norandalign", false);
		args.useStridedAccess = recvTree.getBool("strided", false);
		// extensions of this build (ignored by a reference service)
		args.randOffsetSeed = recvTree.getU64("b200_randseed", 0);
		args.blockVarianceSeed = recvTree.getU64("b200_blockvarseed", 0);
		args.randomVerifySeed = recvTree.getU64("b200_verifyrand", 0);
		args.randomVerifyGrain = recvTree.getU64("b200_verifyrandgrain", 0);
		args.dedupePercent = recvTree.getU64("b200_dedupepct", 0);
		args.pipelineBatchBlocks = recvTree.getU64("b200_batchblocks", 0);
		args.pipelineNumBatches = recvTree.getU64("b200_numbatches", 0);
		args.serializeBufferedWrites = recvTree.getBool("b200_writegate", false);
		args.neverSerializeBufferedWrites = recvTree.getBool("b200_nowritegate", false);
		args.stagingEngineStr = recvTree.getStr("b200_staging", "");
		args.noGPUNumaBinding = recvTree.getBool("b200_nogpunuma", false);
		args.useNoFDSharing = recvTree.getBool("nofdsharing", false);

		const uint64_t numDataSetThreads = recvTree.getU64("datasetthreads", args.numThreads);

		isRWMixConfig = (args.rwMixReadPercent || args.numRWMixReadThreads);

		if(recvTree.getBool("mmap", false) || recvTree.getBool("hdfs", false) ||
			recvTree.getBool("netbench", false) || !recvTree.getStr("s3endpoints", "").empty() )
			throw ProgError("This service is the GPU worker build: mmap, HDFS, S3 and netbench "
				"modes are not available.");

		/* custom tree mode: the file was uploaded to our tmp dir under the given name before
		   (ProgArgs.cpp:3685-3698) */
		args.treeFilePath = recvTree.getStr("treefile", "");

		if(!args.treeFilePath.empty() )
		{
			const size_t slashPos = args.treeFilePath.find_last_of('/');

			if(slashPos != std::string::npos)
				args.treeFilePath = args.treeFilePath.substr(slashPos + 1);

			args.treeFilePath = uploadBasePath() + "/" + args.treeFilePath;
		}

		args.useCustomTreeRandomize = recvTree.getBool("treerand", false);
		args.treeRoundUpSize = recvTree.getU64("treeroundup", 0);
		args.fileShareSize = recvTree.getU64("sharesize", 0);

		if(args.gpuIDsStr.empty() )
			throw ProgError("This service is the GPU worker build: the master has to give "
				"\"--gpuids\" (the on-GPU block fill/verify has no CPU fallback).");

		if(args.integrityCheckSalt)
			args.blockVariancePercent = 0; // ProgArgs.cpp:1161-1167

		// paths: parseAndCheckPaths (ProgArgs.cpp:1683-1745)
		benchPaths.clear();
		size_t start = 0;
		while(start <= benchPathStr.size() )
		{
			size_t delimPos = benchPathStr.find_first_of(ELB_BENCHPATH_DELIMITER, start);
			std::string path = benchPathStr.substr(start,
				(delimPos == std::string::npos) ? std::string::npos : (delimPos - start) );

			if(!path.empty() )
				benchPaths.push_back(path);

			if(delimPos == std::string::npos)
				break;

			start = delimPos + 1;
		}

		if(benchPaths.empty() )
			throw ProgError("Benchmark path missing.");

		args.benchPaths = benchPaths;

		// path type from the first path (ProgArgs::findBenchPathType)
		{
			struct stat statBuf;
			if(stat(benchPaths[0].c_str(), &statBuf) == -1)
				args.benchPathType = ELB_PATH_FILE;
			else
			if(S_ISDIR(statBuf.st_mode) )
				args.benchPathType = ELB_PATH_DIR;
			else
			if(S_ISBLK(statBuf.st_mode) )
				args.benchPathType = ELB_PATH_BLOCKDEV;
			else
				args.benchPathType = ELB_PATH_FILE;
		}

		args.gpuIDs.clear();
		if(args.gpuIDsStr == "all")
		{
			int numGPUs = 0;
			if( (cudaGetDeviceCount(&numGPUs) != cudaSuccess) || !numGPUs)
				throw ProgError("No GPUs found for \"--gpuids all\".");

			for(int gpuID = 0; gpuID < numGPUs; gpuID++)
				args.gpuIDs.push_back(gpuID);
		}
		else
			args.gpuIDs = ProgArgs::parseGPUIDs(args.gpuIDsStr);

		args.toABIConfig(abiConfig);
		abiConfig.cfg.numDataSetThreads = (uint32_t)numDataSetThreads;
		abiConfig.cfg.runAsService = 1;

		manager.reset(new Manager(&abiConfig.cfg) );

		/* workers on several GPUs: create the NCCL communicators of the statistics reduce now,
		   while the workers are idle (and before any result output) */
		if(manager->getNumGPUs() >= 2)
			manager->getLiveReduceInfo();

		// normalised values go back to the master (ProgArgs::getBenchPathInfoTree :3986-3994)
		args.blockSize = manager->shared.cfg.blockSize;
		args.fileSize = manager->shared.cfg.fileSize;
		args.randomAmount = manager->shared.cfg.randomAmount;

		if(!args.benchLabel.empty() )
			std::cout << "LABEL: " << args.benchLabel << std::endl;

		std::cout << std::endl;

		JsonTree replyTree;
		replyTree.put("path", benchPathStr);
		replyTree.put("BenchPathType", (uint64_t)args.benchPathType);
		replyTree.put("NumBenchPaths", (uint64_t)benchPaths.size() );
		replyTree.put("size", args.fileSize);
		replyTree.put("block", args.blockSize);
		replyTree.put("randamount", args.randomAmount);
		replyTree.put("ErrorHistory", errHistory);

		currentPhase = ELB_PHASE_IDLE;
		currentBenchID.clear();

		response.body = replyTree.toJSON();
	}
	catch(std::exception& e)
	{
		resetManager();

		response.statusCode = 400;
		response.body = std::string("Preparation phase error: ") + e.what() + "\n";

		std::cerr << response.body;
	}

	return response;
}

HttpResponse Service::handleStartPhase(const HttpRequest& request)
{
	HttpResponse response;

	if(!request.query.count("PhaseCode") )
	{
		response.statusCode = 400;
		response.body = "Missing parameter: PhaseCode";
		return response;
	}

	const int benchPhase = atoi(request.query.at("PhaseCode").c_str() );
	const std::string benchID = request.query.count("BenchID") ? request.query.at("BenchID") : "";

	if(!manager)
	{
		response.body = "Refusing start request: no benchmark phase was prepared.";
		return response;
	}

	// flaky network: the same start command may arrive twice (HTTPServiceSWS.cpp:534-545)
	if(!benchID.empty() && (benchID == currentBenchID) )
		return response;

	{
		std::unique_lock<std::mutex> lock(manager->shared.mutex);

		if(manager->shared.numWorkersDone != manager->shared.workers.size() )
		{
			response.body = "Refusing start request while not all workers are idle/done. "
				"BenchID: " + benchID + "; "
				"WorkersTotal: " + std::to_string(manager->shared.workers.size() ) + "; "
				"WorkersDoneTotal: " + std::to_string(manager->shared.numWorkersDone) + "\n";
			return response; // non-empty response makes the master's RemoteWorker error out
		}
	}

	liveCpuUtil.update();

	currentBenchID = benchID;
	currentPhase = benchPhase;
	phaseStartT = Clock::now();

	try
	{
		manager->startNextPhase(benchPhase);
	}
	catch(std::exception& e)
	{
		errHistory += std::string("ERROR: ") + e.what() + "\n";
	}

	response.body = errHistory;
	return response;
}

HttpResponse Service::handleInterruptPhase(const HttpRequest& request)
{
	HttpResponse response;

	collectErrHistory();
	resetManager();

	response.body = errHistory;

	if(request.query.count("quit") )
	{
		std::cout << "Shutting down as requested by client. Client: " << request.remoteAddr <<
			std::endl;
		quitRequested = true;
	}

	return response;
}

HttpResponse Service::handle(const HttpRequest& request)
{
	if(progArgs.logLevel > 0)
		std::cout << "HTTP: " << request.method << " " << request.path << std::endl;

	if( (request.path == "/info") && (request.method == "GET") )
	{
		HttpResponse response;
		response.body = "elbencho-b200 service (GPU worker build); protocol "
			ELB_HTTP_PROTOCOLVERSION "\n";
		return response;
	}

	if( (request.path == "/protocolversion") && (request.method == "GET") )
	{
		HttpResponse response;
		response.body = ELB_HTTP_PROTOCOLVERSION;
		return response;
	}

	if( (request.path == "/status") && (request.method == "GET") )
		return handleStatus();

	if( (request.path == "/benchresult") && (request.method == "GET") )
		return handleBenchResult();

	if( (request.path == "/preparephase") && (request.method == "POST") )
		return handlePreparePhase(request);

	if( (request.path == "/preparefile") && (request.method == "POST") )
		return handlePrepareFile(request);

	if( (request.path == "/startphase") && (request.method == "GET") )
		return handleStartPhase(request);

	if( (request.path == "/interruptphase") && (request.method == "GET") )
		return handleInterruptPhase(request);

	HttpResponse response;
	response.statusCode = 404;
	response.body = "Unknown resource: " + request.path;
	return response;
}

/* HTTPServiceSWS::startServer (:29-190): daemonise unless --foreground, then serve */
int Service::run()
{
	int listenSock = socket(AF_INET6, SOCK_STREAM, 0);
	bool isV6 = (listenSock != -1);

	if(!isV6)
		listenSock = socket(AF_INET, SOCK_STREAM, 0);

	if(listenSock == -1)
		throw ProgError(std::string("Unable to create listening socket. SysErr: ") +
			strerror(errno) );

	int enable = 1;
	setsockopt(listenSock, SOL_SOCKET, SO_REUSEADDR, &enable, sizeof(enable) );

	int bindRes;

	if(isV6)
	{
		int disable = 0;
		setsockopt(listenSock, IPPROTO_IPV6, IPV6_V6ONLY, &disable, sizeof(disable) );

		struct sockaddr_in6 addr;
		memset(&addr, 0, sizeof(addr) );
		addr.sin6_family = AF_INET6;
		addr.sin6_addr = in6addr_any;
		addr.sin6_port = htons( (unsigned short)progArgs.servicePort);
		bindRes = bind(listenSock, (struct sockaddr*)&addr, sizeof(addr) );
	}
	else
	{
		struct sockaddr_in addr;
		memset(&addr, 0, sizeof(addr) );
		addr.sin_family = AF_INET;
		addr.sin_addr.s_addr = htonl(INADDR_ANY);
		addr.sin_port = htons( (unsigned short)progArgs.servicePort);
		bindRes = bind(listenSock, (struct sockaddr*)&addr, sizeof(addr) );
	}

	if(bindRes == -1)
	{
		int bindErrno = errno;
		close(listenSock);
		throw ProgError("Unable to bind to desired port. Port: " +
			std::to_string(progArgs.servicePort) + "; SysErr: " + strerror(bindErrno) );
	}

	if(listen(listenSock, 128) == -1)
	{
		close(listenSock);
		throw ProgError(std::string("Unable to listen on socket. SysErr: ") + strerror(errno) );
	}

	if(!progArgs.runServiceInForeground)
	{ // daemonize (HTTPServiceSWS.cpp:45-110): log goes to a file in /tmp
		const std::string logFile = "/tmp/elbencho-b200_" + std::to_string(getuid() ) + "_p" +
			std::to_string(progArgs.servicePort) + ".log";

		std::cout << "Daemonizing into background... Logfile: " << logFile << std::endl;

		pid_t childPID = fork();

		if(childPID == -1)
			throw ProgError(std::string("Unable to fork. SysErr: ") + strerror(errno) );

		if(childPID > 0)
			_exit(EXIT_SUCCESS); // parent: the service lives on in the child

		setsid();

		int logFD = open(logFile.c_str(), O_CREAT | O_WRONLY | O_TRUNC, 0644);
		int nullFD = open("/dev/null", O_RDONLY);

		if(logFD != -1)
		{
			dup2(logFD, STDOUT_FILENO);
			dup2(logFD, STDERR_FILENO);
			close(logFD);
		}

		if(nullFD != -1)
		{
			dup2(nullFD, STDIN_FILENO);
			close(nullFD);
		}
	}

	signal(SIGPIPE, SIG_IGN);

	std::cout << "Elbencho-b200 service now listening. Port: " << progArgs.servicePort <<
		std::endl;

	struct Connection
	{
		int sock;
		std::string buffer;
		std::string remoteAddr;
		size_t neededLen{0}; // known size of the message being received (0 = headers not seen)
	};

	std::vector<Connection> connections;

	while(!quitRequested)
	{
		std::vector<struct pollfd> pollFDs;
		pollFDs.push_back( {listenSock, POLLIN, 0} );

		for(const Connection& conn : connections)
			pollFDs.push_back( {conn.sock, POLLIN, 0} );

		int pollRes = poll(pollFDs.data(), pollFDs.size(), 1000);

		if(pollRes < 0)
		{
			if(errno == EINTR)
				continue;

			break;
		}

		if(pollFDs[0].revents & POLLIN)
		{
			struct sockaddr_storage peerAddr;
			socklen_t peerLen = sizeof(peerAddr);
			int sock = accept(listenSock, (struct sockaddr*)&peerAddr, &peerLen);

			if(sock != -1)
			{
				int noDelay = 1;
				setsockopt(sock, IPPROTO_TCP, TCP_NODELAY, &noDelay, sizeof(noDelay) );

				char hostBuf[NI_MAXHOST] = "";
				getnameinfo( (struct sockaddr*)&peerAddr, peerLen, hostBuf, sizeof(hostBuf), NULL,
					0, NI_NUMERICHOST);

				connections.push_back( {sock, "", hostBuf} );
			}
		}

		// (index into connections = poll index - 1; iterate backwards so erase is safe)
		for(size_t pollIdx = pollFDs.size() - 1; pollIdx >= 1; pollIdx--)
		{
			if(!(pollFDs[pollIdx].revents & (POLLIN | POLLHUP | POLLERR) ) )
				continue;

			Connection& conn = connections[pollIdx - 1];
			char chunk[65536];
			ssize_t recvRes = recv(conn.sock, chunk, sizeof(chunk), 0);

			bool closeConn = (recvRes <= 0);

			if(recvRes > 0)
			{
				conn.buffer.append(chunk, recvRes);

				if(conn.buffer.size() > ELB_HTTP_MAX_REQUEST_BYTES)
					closeConn = true;
			}

			while(!closeConn)
			{
				/* (the headers are parsed once per message, not once per received chunk: the rest
				   of a large upload is only appended) */
				if(conn.neededLen && (conn.buffer.size() < conn.neededLen) )
					break;

				HttpMessageView view = parseHttpMessage(conn.buffer, false, false);

				if(view.invalid)
				{
					closeConn = true;
					break;
				}

				conn.neededLen = view.complete ? 0 : view.neededLen;

				if(!view.complete)
					break;

				HttpRequest request;
				request.remoteAddr = conn.remoteAddr;
				request.body = view.body;

				std::stringstream startLineStream(view.startLine);
				std::string target;
				startLineStream >> request.method >> target;

				const size_t queryPos = target.find('?');
				request.path = target.substr(0, queryPos);

				if(queryPos != std::string::npos)
					parseQuery(target.substr(queryPos + 1), request.query);

				HttpResponse response = handle(request);

				std::string connHeader = view.headers.count("connection") ?
					view.headers["connection"] : "";
				std::transform(connHeader.begin(), connHeader.end(), connHeader.begin(),
					::tolower);
				const bool keepAlive = (connHeader != "close") && !quitRequested;

				std::string reply = "HTTP/1.1 " + std::to_string(response.statusCode) + " " +
					httpStatusText(response.statusCode) + "\r\n"
					"Content-Length: " + std::to_string(response.body.size() ) + "\r\n" +
					(keepAlive ? "" : "Connection: close\r\n") + "\r\n" + response.body;

				if(!sendAll(conn.sock, reply) || !keepAlive)
					closeConn = true;

				conn.buffer.erase(0, view.totalLen);
			}

			if(closeConn)
			{
				close(conn.sock);
				connections.erase(connections.begin() + (pollIdx - 1) );
			}
		}
	}

	for(const Connection& conn : connections)
		close(conn.sock);

	close(listenSock);
	resetManager();

	return EXIT_SUCCESS;
}

int serviceMain(ProgArgs& progArgs)
{
	Service service(progArgs);
	return service.run();
}

/* ==============================================================================================
 * Master side (RemoteWorker.cpp + the coordinator parts that differ in master mode)
 * ============================================================================================ */

struct RemoteHost
{
	std::string host;
	unsigned short port;
	size_t numWorkersDone{0};
	size_t numWorkersDoneWithError{0};
	elb_liveops liveOps{};
	elb_liveops liveOpsReadMix{};
	elb_liveops stoneWallOps{};
	elb_liveops stoneWallOpsReadMix{};
	bool gotPhaseWork{true};
	bool isDone{false};
	std::vector<uint64_t> elapsedUSecVec;
	elb_histogram iopsLatHisto, entriesLatHisto, iopsLatHistoReadMix, entriesLatHistoReadMix;
	unsigned cpuUtilStoneWall{0}, cpuUtilLastDone{0}, cpuUtilLive{0};
	elb_livelat liveLat{}; // sums of the status replies since the last live CSV line
	std::string errorMsg;
};

static void splitHostPort(const std::string& hostStr, unsigned short defaultPort,
	std::string& outHost, unsigned short& outPort)
{ // RemoteWorker: "host[:port]"
	const size_t colonPos = hostStr.rfind(':');

	if( (colonPos == std::string::npos) || (hostStr.find(']') != std::string::npos) )
	{
		outHost = hostStr;
		outPort = defaultPort;
		return;
	}

	outHost = hostStr.substr(0, colonPos);
	outPort = (unsigned short)atoi(hostStr.c_str() + colonPos + 1);
}

/* hosts with square bracket ranges, e.g. "localhost:[1711-1712]" or "node[01-04]"
 * (TranslatorTk::splitAndExpandStr, toolkits/TranslatorTk.cpp:611-633) */
static std::vector<std::string> expandHosts(const std::vector<std::string>& hosts)
{
	std::vector<std::string> expanded;

	for(const std::string& host : hosts)
	{
		const size_t openPos = host.find('[');
		const size_t closePos = host.find(']');
		const size_t dashPos = host.find('-', (openPos == std::string::npos) ? 0 : openPos);

		if( (openPos == std::string::npos) || (closePos == std::string::npos) ||
			(dashPos == std::string::npos) || (dashPos > closePos) )
		{
			expanded.push_back(host);
			continue;
		}

		const std::string firstStr = host.substr(openPos + 1, dashPos - openPos - 1);
		const std::string lastStr = host.substr(dashPos + 1, closePos - dashPos - 1);
		const long first = atol(firstStr.c_str() );
		const long last = atol(lastStr.c_str() );

		for(long value = first; value <= last; value++)
		{
			std::string valueStr = std::to_string(value);

			if( (firstStr.size() > 1) && (firstStr[0] == '0') && (valueStr.size() < firstStr.size() ) )
				valueStr = std::string(firstStr.size() - valueStr.size(), '0') + valueStr;

			expanded.push_back(host.substr(0, openPos) + valueStr + host.substr(closePos + 1) );
		}
	}

	return expanded;
}

static std::string generateBenchID()
{ // boost::uuids::random_generator text form
	std::random_device randDev;
	char buf[40];

	snprintf(buf, sizeof(buf), "%08x-%04x-4%03x-%04x-%08x%04x", randDev(), randDev() & 0xffff,
		randDev() & 0xfff, (randDev() & 0x3fff) | 0x8000, randDev(), randDev() & 0xffff);

	return buf;
}

/* ProgArgs::getAsPropertyTreeForService (ProgArgs.cpp:3725-3863): every key the reference puts,
 * with the values of the supported subset and neutral values for the rest */
static JsonTree progArgsToServiceTree(const ProgArgs& args, size_t serviceRank, size_t numHosts)
{
	JsonTree tree;
	std::string benchPathStr;

	for(const std::string& path : args.benchPaths)
	{
		std::string absPath = path;

		if(!path.empty() && (path[0] != '/') )
		{
			char cwdBuf[4096];
			if(getcwd(cwdBuf, sizeof(cwdBuf) ) )
				absPath = std::string(cwdBuf) + "/" + path;
		}

		benchPathStr += absPath + ",";
	}

	tree.put("block", args.blockSize);
	tree.put("blockvarpct", args.blockVariancePercent);
	tree.put("blockvaralgo", args.blockVarianceAlgo.empty() ? "fast" : args.blockVarianceAlgo);
	tree.put("label", args.benchLabel);
	tree.put("benchmode", (uint64_t)1); // BenchMode_POSIX (Common.h:130-137)
	tree.put("path", benchPathStr);
	tree.putBool("mkdirs", args.runCreateDirsPhase);
	tree.putBool("write", args.runCreateFilesPhase);
	tree.putBool("cufile", args.useCuFile);
	tree.putBool("cufiledriveropen", false);
	tree.putBool("cuhostbufreg", false);
	tree.putBool("deldirs", args.runDeleteDirsPhase);
	tree.putBool("delfiles", args.runDeleteFilesPhase);
	tree.putBool("dirsharing", args.doDirSharing);
	tree.putBool("direct", args.useDirectIO);
	tree.putBool("dropcache", args.runDropCachesPhase);
	tree.put("fadv", args.fadviseFlags);
	tree.put("sharesize", args.fileShareSize);
	tree.put("size", args.fileSize);
	tree.put("flock", args.flockType);
	tree.putBool("gdsbufreg", args.useGDSBufReg);
	tree.putBool("hdfs", false);
	tree.putBool("no0usecerr", args.ignore0USecErrors);
	tree.putBool("nodelerr", args.ignoreDelErrors);
	tree.putBool("infloop", args.doInfiniteIOLoop);
	tree.put("b200_timelimit", args.timeLimitSecs); // (applied by the service at /status time)
	tree.put("verify", args.integrityCheckSalt);
	tree.put("iodepth", args.ioDepth);
	tree.put("limitread", args.limitReadBps);
	tree.put("limitwrite", args.limitWriteBps);
	tree.put("madv", (uint64_t)0);
	tree.putBool("mmap", false);
	tree.putBool("netbench", false);
	tree.put("netbenchservers", "");
	// (services that do not share their paths each work on a full data set, ProgArgs.cpp:1288)
	tree.put("datasetthreads", args.noSharedServicePath ?
		args.numThreads : (args.numThreads * numHosts) );
	tree.put("dirs", args.numDirs);
	tree.put("files", args.numFiles);
	tree.put("numservers", (uint64_t)0);
	tree.put("threads", args.numThreads);
	tree.putBool("nofdsharing", args.useNoFDSharing);
	tree.putBool("nodiocheck", args.noDirectIOCheck);
	tree.putBool("opsloglock", false);
	tree.put("opslog", "");
	tree.putBool("preallocfile", args.doPreallocFile);
	tree.putBool("norandalign", args.useRandomUnaligned);
	tree.put("randamount", args.randomAmount);
	tree.putBool("rand", args.useRandomOffsets);
	tree.put("randalgo", args.randOffsetAlgo);
	tree.putBool("read", args.runReadPhase);
	tree.putBool("readinline", args.doReadInline);
	tree.put("recvbuf", (uint64_t)0);
	tree.put("respsize", (uint64_t)1);
	tree.putBool("backward", args.doReverseSeqOffsets);
	tree.put("rwmixpct", args.rwMixReadPercent);
	tree.put("rwmixthr", args.numRWMixReadThreads);
	tree.put("rwmixthrpct", args.rwMixThreadsReadPercent);

	// S3 keys: neutral values
	const char* s3EmptyStrings[] = {"s3key", "s3secret", "s3aclgrantee", "s3aclgtype",
		"s3aclgrants", "s3chksumalgo", "s3credfile", "s3credlist", "s3endpoints", "s3objprefix",
		"s3region", "s3sessiontoken", "s3sseckey", "s3ssekmskey"};
	for(const char* key : s3EmptyStrings)
		tree.put(key, "");

	const char* s3FalseFlags[] = {"s3aclget", "s3aclput", "s3aclputinl", "s3aclverify",
		"s3baclget", "s3baclput", "s3btag", "s3btagverify", "s3bversion", "s3bversionverify",
		"s3single", "s3fastget", "s3ignoreerrors", "s3listobjpar", "s3listverify",
		"s3multiignore404", "s3nocompress", "s3nompucompl", "s3olockcfg", "s3olockcfgverify",
		"s3otag", "s3otagverify", "s3randobj", "s3sse", "s3statdirs", "s3virtaddr"};
	for(const char* key : s3FalseFlags)
		tree.putBool(key, false);

	const char* s3Zeros[] = {"s3listobj", "s3maxconns", "s3mpusizevar", "s3mpusplit",
		"s3multidel", "s3sign", "s3targetgbps"};
	for(const char* key : s3Zeros)
		tree.put(key, (uint64_t)0);

	tree.put("sendbuf", (uint64_t)0);
	tree.putBool("stat", args.runStatFilesPhase);
	tree.putBool("statinline", args.doStatInline);
	tree.putBool("strided", args.useStridedAccess);
	tree.putBool("sync", args.runSyncPhase);
	tree.putBool("trunc", args.doTruncate);
	tree.putBool("trunctosize", args.doTruncToSize);
	tree.putBool("treerand", args.useCustomTreeRandomize);
	tree.put("treeroundup", args.treeRoundUpSize);
	tree.putBool("verifydirect", args.doDirectVerify);

	// dynamically calculated values for service hosts (:3845-3861)
	tree.put("rankoffset", args.noSharedServicePath ?
		args.rankOffset : (args.rankOffset + (serviceRank * args.numThreads) ) );
	tree.put("treefile", args.treeFilePath.empty() ? "" : "treefile.txt"); // ProgArgs.cpp:3850
	if(!args.assignGPUPerService || args.gpuIDs.empty() )
		tree.put("gpuids", args.gpuIDsStr);
	else
	{ // --gpuperservice: one GPU of the list per service instance (ProgArgs.cpp:3852-3859)
		const size_t gpuIndex = serviceRank % args.gpuIDs.size();
		tree.put("gpuids", std::to_string(args.gpuIDs[gpuIndex] ) );
	}

	// extensions of this build
	tree.put("b200_randseed", args.randOffsetSeed);
	tree.put("b200_blockvarseed", args.blockVarianceSeed);
	tree.put("b200_verifyrand", args.randomVerifySeed);
	tree.put("b200_verifyrandgrain", args.randomVerifyGrain);
	tree.put("b200_dedupepct", args.dedupePercent);
	tree.put("b200_batchblocks", args.pipelineBatchBlocks);
	tree.put("b200_numbatches", args.pipelineNumBatches);
	tree.putBool("b200_writegate", args.serializeBufferedWrites);
	tree.putBool("b200_nowritegate", args.neverSerializeBufferedWrites);
	tree.put("b200_staging", args.stagingEngineStr);
	tree.putBool("b200_nogpunuma", args.noGPUNumaBinding);

	return tree;
}

class Master
{
	public:
		explicit Master(ProgArgs& progArgs) : progArgs(progArgs) {}

		int run();
		int interruptOrQuit();

	private:
		ProgArgs& progArgs;
		std::vector<RemoteHost> hosts;
		uint64_t phaseCounter{0};

		void initHosts();
		void prepareRemotePhases();
		void runPhase(int benchPhase);
		void runSyncAndDropCaches();
		void interruptAll(bool quit);
		void waitForServicesReady();
		void rotateHosts();
		void getExpectedTotals(int benchPhase, uint64_t& outEntries, uint64_t& outBytes);
		void printLiveStatsCSV(int benchPhase, elb_liveops oldLiveOps[2],
			Clock::time_point& lastT, const Clock::time_point& phaseStartT,
			uint64_t expectedEntries, uint64_t expectedBytes);
		bool liveCSVHeaderPrinted{false};
		bool isPhaseTimeExpired{false};
};

void Master::initHosts()
{
	for(const std::string& hostStr : expandHosts(progArgs.hosts) )
	{
		RemoteHost remote;
		splitHostPort(hostStr, (unsigned short)progArgs.servicePort, remote.host, remote.port);
		hosts.push_back(remote);
	}

	if(hosts.empty() )
		throw ProgError("Hosts list is empty.");
}

/* RemoteWorker::preparePhase (RemoteWorker.cpp:270-350): POST /preparephase on every service in
 * parallel, check the returned BenchPathInfo for consistency (ProgArgs.cpp:4004-4080) */
void Master::prepareRemotePhases()
{
	std::vector<std::thread> threads;
	std::vector<JsonTree> replies(hosts.size() );

	for(size_t i = 0; i < hosts.size(); i++)
		threads.emplace_back([this, i, &replies]()
		{
			RemoteHost& remote = hosts[i];

			try
			{
				if(!progArgs.treeFilePath.empty() )
				{ // RemoteWorker::prepareRemoteFile (RemoteWorker.cpp:286-330)
					std::ifstream treeFileStream(progArgs.treeFilePath);

					if(!treeFileStream)
						throw ProgError("Unable to read custom tree file. Path: " +
							progArgs.treeFilePath);

					std::stringstream treeFileContents;
					treeFileContents << treeFileStream.rdbuf();

					HttpResponse uploadResponse = httpRequest(remote.host, remote.port, "POST",
						"/preparefile?ProtocolVersion=" ELB_HTTP_PROTOCOLVERSION
						"&FileName=treefile.txt&PwHash=" + progArgs.svcPasswordHash,
						treeFileContents.str(), 60);

					if(uploadResponse.statusCode != 200)
						throw ProgError("Service encountered an error. Service: " + remote.host +
							":" + std::to_string(remote.port) + "; Phase: File preparation; "
							"Message: " + uploadResponse.body);
				}

				JsonTree tree = progArgsToServiceTree(progArgs, i, hosts.size() );

				HttpResponse response = httpRequest(remote.host, remote.port, "POST",
					"/preparephase?ProtocolVersion=" ELB_HTTP_PROTOCOLVERSION "&PwHash=" +
						progArgs.svcPasswordHash,
					tree.toJSON(), 300);

				if(response.statusCode != 200)
					throw ProgError("Service encountered an error. Service: " + remote.host + ":" +
						std::to_string(remote.port) + "; Phase: Preparation; Message: " +
						response.body);

				replies[i] = JsonTree::parse(response.body);
			}
			catch(std::exception& e)
			{
				remote.errorMsg = e.what();
			}
		});

	for(std::thread& thread : threads)
		thread.join();

	for(const RemoteHost& remote : hosts)
		if(!remote.errorMsg.empty() )
			throw ProgError(remote.errorMsg);

	// all services have to agree on path type, sizes (checkServiceBenchPathInfos)
	for(size_t i = 0; i < hosts.size(); i++)
	{
		const JsonTree& reply = replies[i];

		if( (reply.getU64("BenchPathType") != replies[0].getU64("BenchPathType") ) ||
			(reply.getU64("size") != replies[0].getU64("size") ) ||
			(reply.getU64("block") != replies[0].getU64("block") ) )
			throw ProgError("Conflicting benchmark path info from services. "
				"Service A: " + hosts[0].host + "; Service B: " + hosts[i].host);

		const std::string remoteErrHistory = reply.getStr("ErrorHistory", "");
		if(!remoteErrHistory.empty() )
			std::cerr << "[" << hosts[i].host << "] " << remoteErrHistory;
	}

	progArgs.benchPathType = (int)replies[0].getU64("BenchPathType");
	progArgs.fileSize = replies[0].getU64("size");
	progArgs.blockSize = replies[0].getU64("block");
	progArgs.randomAmount = replies[0].getU64("randamount");
}

void Master::interruptAll(bool quit)
{
	for(RemoteHost& remote : hosts)
	{
		try
		{
			httpRequest(remote.host, remote.port, "GET",
				quit ? "/interruptphase?quit" : "/interruptphase", "", 60);
		}
		catch(std::exception& e)
		{
			std::cerr << "ERROR: " << e.what() << std::endl;
		}
	}
}

/* one phase on all services: RemoteWorker::startBenchPhase / waitForBenchPhaseCompletion /
 * finishPhase (RemoteWorker.cpp:352-572, 169-268) and the master side of
 * Statistics::generatePhaseResults */
void Master::runPhase(int benchPhase)
{
	if(isPhaseTimeExpired) // Coordinator::checkInterruptionBetweenPhases (Coordinator.cpp:234-241)
		throw ProgTimeLimit();

	const std::string benchID = generateBenchID();
	const Clock::time_point phaseStartT = Clock::now();
	const bool isRWMixConfig = (progArgs.rwMixReadPercent || progArgs.numRWMixReadThreads) &&
		(benchPhase == ELB_PHASE_CREATEFILES);

	phaseCounter++;

	char isoBuf[64];
	{
		time_t nowSecs = time(NULL);
		struct tm localTimeInfo;
		localtime_r(&nowSecs, &localTimeInfo);
		strftime(isoBuf, sizeof(isoBuf), "%FT%T.000%z", &localTimeInfo);
	}

	for(RemoteHost& remote : hosts)
	{
		remote = RemoteHost{remote.host, remote.port};
		histogramReset(remote.iopsLatHisto);
		histogramReset(remote.entriesLatHisto);
		histogramReset(remote.iopsLatHistoReadMix);
		histogramReset(remote.entriesLatHistoReadMix);

		HttpResponse response = httpRequest(remote.host, remote.port, "GET",
			"/startphase?PhaseCode=" + std::to_string(benchPhase) + "&BenchID=" + benchID, "", 60);

		if( (response.statusCode != 200) || !response.body.empty() )
			throw ProgError("Service encountered an error. Service: " + remote.host + "; "
				"Phase: Benchmark start; Message: " + response.body);
	}

	bool stoneWallTaken = false;
	elb_liveops oldLiveOps{};
	elb_liveops oldLiveOpsCSV[2] = {};
	Clock::time_point lastLiveCSVT = phaseStartT;
	uint64_t expectedEntries = 0, expectedBytes = 0;

	if(!progArgs.liveCSVFilePath.empty() )
		getExpectedTotals(benchPhase, expectedEntries, expectedBytes);

	Clock::time_point lastLiveT = phaseStartT;
	bool printedLiveLine = false;
	const bool showLive = !progArgs.disableLiveStats && isatty(STDOUT_FILENO);

	for( ; ; )
	{
		std::this_thread::sleep_for(std::chrono::milliseconds(
			progArgs.svcUpdateIntervalMS ? progArgs.svcUpdateIntervalMS : ELB_SVC_UPDATE_INTERVAL_MS) );

		size_t numHostsDone = 0;

		for(RemoteHost& remote : hosts)
		{
			if(remote.isDone)
			{
				numHostsDone++;
				continue;
			}

			HttpResponse response = httpRequest(remote.host, remote.port, "GET", "/status", "", 60);

			if(response.statusCode != 200)
				throw ProgError("Service encountered an error. Service: " + remote.host + "; "
					"Phase: Wait for benchmark completion; HTTP status code: " +
					std::to_string(response.statusCode) );

			JsonTree statusTree = JsonTree::parse(response.body);

			if(statusTree.getStr("BenchID") != benchID)
				throw ProgError("Service got hijacked for a different benchmark. Service: " +
					remote.host);

			remote.numWorkersDone = statusTree.getU64("NumWorkersDone");
			remote.numWorkersDoneWithError = statusTree.getU64("NumWorkersDoneWithError");
			remote.liveOps.numEntriesDone = statusTree.getU64("NumEntriesDone");
			remote.liveOps.numBytesDone = statusTree.getU64("NumBytesDone");
			remote.liveOps.numIOPSDone = statusTree.getU64("NumIOPSDone");
			remote.cpuUtilLive = (unsigned)statusTree.getU64("CPUUtil", 0);
			remote.liveLat.numAvgIOLatValues += statusTree.getU64("NumIOLatUSec", 0);
			remote.liveLat.avgIOLatMicroSecsSum += statusTree.getU64("SumIOLatUSec", 0);
			remote.liveLat.numAvgEntriesLatValues += statusTree.getU64("NumEntLatUSec", 0);
			remote.liveLat.avgEntriesLatMicroSecsSum += statusTree.getU64("SumEntLatUSec", 0);

			if(isRWMixConfig)
			{
				remote.liveOpsReadMix.numEntriesDone = statusTree.getU64("NumEntriesDoneRWMixRead", 0);
				remote.liveOpsReadMix.numBytesDone = statusTree.getU64("NumBytesDoneRWMixRead", 0);
				remote.liveOpsReadMix.numIOPSDone = statusTree.getU64("NumIOPSDoneRWMixRead", 0);
			}

			if(remote.numWorkersDoneWithError)
				throw ProgError("[" + remote.host + "] " + statusTree.getStr("ErrorHistory", "") );

			if(remote.numWorkersDone >= progArgs.numThreads)
			{
				remote.isDone = true;
				numHostsDone++;
			}

			/* stonewall: when the first service with work is done, snapshot the live ops of all
			   services (RemoteWorker::createStoneWallStats through Worker::incNumWorkersDone) */
			if(!stoneWallTaken && statusTree.getBool("TriggerStoneWall", false) )
			{
				stoneWallTaken = true;

				for(RemoteHost& other : hosts)
				{
					other.stoneWallOps = other.liveOps;
					other.stoneWallOpsReadMix = other.liveOpsReadMix;
				}
			}
		}

		if(numHostsDone == hosts.size() )
			break;

		if(!progArgs.liveCSVFilePath.empty() )
			printLiveStatsCSV(benchPhase, oldLiveOpsCSV, lastLiveCSVT, phaseStartT, expectedEntries,
				expectedBytes);

		if(showLive)
		{
			elb_liveops liveOps{};
			for(const RemoteHost& remote : hosts)
				liveOpsAdd(liveOps, remote.liveOps);

			const Clock::time_point nowT = Clock::now();
			const uint64_t intervalUSec =
				std::chrono::duration_cast<std::chrono::microseconds>(nowT - lastLiveT).count();
			const uint64_t mib = 1024 * 1024;

			std::cout << "\x1b[2K\r" << stats::phaseName(benchPhase, progArgs) << ": " <<
				perSecFromUSec(liveOps.numIOPSDone - oldLiveOps.numIOPSDone, intervalUSec) <<
				" IOPS; " <<
				perSecFromUSec(liveOps.numBytesDone - oldLiveOps.numBytesDone, intervalUSec) / mib <<
				" MiB/s; " << liveOps.numBytesDone / mib << " MiB; " <<
				(hosts.size() - numHostsDone) << " services; " <<
				std::chrono::duration_cast<std::chrono::seconds>(nowT - phaseStartT).count() <<
				"s" << std::flush;

			printedLiveLine = true;
			oldLiveOps = liveOps;
			lastLiveT = nowT;
		}
	}

	if(printedLiveLine)
		std::cout << "\x1b[2K\r" << std::flush;

	if(progArgs.timeLimitSecs && ( (uint64_t)std::chrono::duration_cast<std::chrono::seconds>(
		Clock::now() - phaseStartT).count() >= progArgs.timeLimitSecs) )
		isPhaseTimeExpired = true;

	// final results of every service (RemoteWorker::finishPhase)
	elb_phase_results res;
	memset(&res, 0, sizeof(res) );
	histogramReset(res.iopsLatHisto);
	histogramReset(res.entriesLatHisto);
	histogramReset(res.iopsLatHistoReadMix);
	histogramReset(res.entriesLatHistoReadMix);

	std::vector<uint64_t> allElapsedUSec;
	uint64_t cpuStoneWallSum = 0, cpuLastDoneSum = 0;

	for(RemoteHost& remote : hosts)
	{
		HttpResponse response = httpRequest(remote.host, remote.port, "GET", "/benchresult", "",
			120);

		if(response.statusCode != 200)
			throw ProgError("Service instance encountered an error. Service: " + remote.host +
				"; Phase: Finalization; Message: " + response.body);

		JsonTree resultTree = JsonTree::parse(response.body);

		if(resultTree.getStr("BenchID") != benchID)
			throw ProgError("Service instance got hijacked for a different benchmark. Service: " +
				remote.host);

		if(resultTree.getU64("NumWorkersDoneWithError") )
			throw ProgError("[" + remote.host + "] " + resultTree.getStr("ErrorHistory", "") );

		remote.gotPhaseWork = resultTree.getBool("TriggerStoneWall");
		remote.liveOps.numEntriesDone = resultTree.getU64("NumEntriesDone");
		remote.liveOps.numBytesDone = resultTree.getU64("NumBytesDone");
		remote.liveOps.numIOPSDone = resultTree.getU64("NumIOPSDone");
		remote.cpuUtilStoneWall = (unsigned)resultTree.getU64("CPUUtilStoneWall", 0);
		remote.cpuUtilLastDone = (unsigned)resultTree.getU64("CPUUtil", 0);

		const JsonTree* elapsedList = resultTree.find("ElapsedUSecList");
		if(elapsedList)
			for(const std::pair<std::string, JsonTree>& item : elapsedList->getChildren() )
				remote.elapsedUSecVec.push_back(strtoull(item.second.getValue().c_str(), NULL, 10) );

		histogramFromTree(resultTree, "IOPS_", remote.iopsLatHisto);
		histogramFromTree(resultTree, "Entries_", remote.entriesLatHisto);

		if(isRWMixConfig)
		{
			remote.liveOpsReadMix.numEntriesDone = resultTree.getU64("NumEntriesDoneRWMixRead", 0);
			remote.liveOpsReadMix.numBytesDone = resultTree.getU64("NumBytesDoneRWMixRead", 0);
			remote.liveOpsReadMix.numIOPSDone = resultTree.getU64("NumIOPSDoneRWMixRead", 0);
			histogramFromTree(resultTree, "IOPSRWMixRead_", remote.iopsLatHistoReadMix);
			histogramFromTree(resultTree, "EntriesRWMixRead_", remote.entriesLatHistoReadMix);
		}

		if(!stoneWallTaken)
		{ // phase was shorter than one poll interval: first done == last done for the ops
			remote.stoneWallOps = remote.liveOps;
			remote.stoneWallOpsReadMix = remote.liveOpsReadMix;
		}

		liveOpsAdd(res.opsTotal, remote.liveOps);
		liveOpsAdd(res.opsReadMixTotal, remote.liveOpsReadMix);
		liveOpsAdd(res.opsStoneWallTotal, remote.stoneWallOps);
		liveOpsAdd(res.opsStoneWallReadMixTotal, remote.stoneWallOpsReadMix);
		histogramMerge(res.iopsLatHisto, remote.iopsLatHisto);
		histogramMerge(res.entriesLatHisto, remote.entriesLatHisto);
		histogramMerge(res.iopsLatHistoReadMix, remote.iopsLatHistoReadMix);
		histogramMerge(res.entriesLatHistoReadMix, remote.entriesLatHistoReadMix);

		allElapsedUSec.insert(allElapsedUSec.end(), remote.elapsedUSecVec.begin(),
			remote.elapsedUSecVec.end() );

		cpuStoneWallSum += remote.cpuUtilStoneWall;
		cpuLastDoneSum += remote.cpuUtilLastDone;
		res.numWorkersDone += (uint32_t)remote.numWorkersDone;
	}

	if(!allElapsedUSec.empty() )
	{
		res.firstFinishUSec = *std::min_element(allElapsedUSec.begin(), allElapsedUSec.end() );
		res.lastFinishUSec = *std::max_element(allElapsedUSec.begin(), allElapsedUSec.end() );
	}

	auto perSec = [](const elb_liveops& total, uint64_t usec, elb_liveops& out)
	{
		if(!usec)
			return;

		out.numEntriesDone = perSecFromUSec(total.numEntriesDone, usec);
		out.numBytesDone = perSecFromUSec(total.numBytesDone, usec);
		out.numIOPSDone = perSecFromUSec(total.numIOPSDone, usec);
	};

	perSec(res.opsTotal, res.lastFinishUSec, res.opsPerSec);
	perSec(res.opsStoneWallTotal, res.firstFinishUSec, res.opsStoneWallPerSec);

	if(res.opsReadMixTotal.numIOPSDone)
	{
		perSec(res.opsReadMixTotal, res.lastFinishUSec, res.opsReadMixPerSec);
		perSec(res.opsStoneWallReadMixTotal, res.firstFinishUSec, res.opsStoneWallReadMixPerSec);
	}

	res.cpuUtilStoneWallPercent = (uint32_t)(cpuStoneWallSum / hosts.size() );
	res.cpuUtilPercent = (uint32_t)(cpuLastDoneSum / hosts.size() );

	if(allElapsedUSec.empty() )
		std::cout << "Skipping stats print due to unavailable worker results." << std::endl;
	else
	{
		// --svcelapsed: slowest thread of each service (Statistics.cpp:2093-2108)
		std::vector<std::pair<uint64_t, std::string> > svcCompletionMS;

		for(const RemoteHost& remote : hosts)
		{
			uint64_t slowestThreadUSec = 0;

			for(uint64_t elapsedUSec : remote.elapsedUSecVec)
				slowestThreadUSec = std::max(slowestThreadUSec, elapsedUSec);

			svcCompletionMS.push_back(std::make_pair(slowestThreadUSec / 1000,
				remote.host + ":" + std::to_string(remote.port) ) );
		}

		stats::printPhaseResults(progArgs, benchPhase, res, allElapsedUSec, std::cout,
			&svcCompletionMS);

		if(!progArgs.resFilePath.empty() )
		{
			std::ofstream fileStream(progArgs.resFilePath, std::ofstream::app);
			stats::printPhaseResults(progArgs, benchPhase, res, allElapsedUSec, fileStream,
				&svcCompletionMS);
			fileStream << std::endl;
		}

		if(!progArgs.csvFilePath.empty() )
		{
			std::vector<std::string> labels, values;
			stats::csvLabelsAndValues(progArgs, benchPhase, res, isoBuf, labels, values);

			bool needLabels = !progArgs.noCSVLabels;
			{
				std::ifstream existing(progArgs.csvFilePath);
				if(existing && (existing.peek() != std::ifstream::traits_type::eof() ) )
					needLabels = false;
			}

			std::ofstream fileStream(progArgs.csvFilePath, std::ofstream::app);

			auto joinCSV = [](const std::vector<std::string>& vec)
			{
				std::string line;
				for(size_t i = 0; i < vec.size(); i++)
					line += (i ? "," : "") + vec[i];
				return line;
			};

			if(needLabels)
				fileStream << joinCSV(labels) << std::endl;

			fileStream << joinCSV(values) << std::endl;
		}

		if(!progArgs.jsonFilePath.empty() )
		{
			std::ofstream fileStream(progArgs.jsonFilePath, std::ofstream::app);
			fileStream << stats::phaseResultsJSON(progArgs, benchPhase, res, phaseCounter,
				isoBuf) << std::endl;
		}
	}
}

void Master::runSyncAndDropCaches()
{
	if(progArgs.runSyncPhase)
		runPhase(ELB_PHASE_SYNC);

	if(progArgs.runDropCachesPhase)
		runPhase(ELB_PHASE_DROPCACHES);
}

/* Coordinator::waitForServicesReady (Coordinator.cpp:160-230): GET /status on every service until
 * all answer or --svcwait seconds are over */
void Master::waitForServicesReady()
{
	if(!progArgs.svcReadyWaitSec)
		return;

	const Clock::time_point endWaitT =
		Clock::now() + std::chrono::seconds(progArgs.svcReadyWaitSec);

	for( ; ; )
	{
		std::string notReadyServiceHost;

		for(const RemoteHost& remote : hosts)
		{
			try
			{
				HttpResponse response = httpRequest(remote.host, remote.port, "GET", "/status", "",
					(int)progArgs.svcReadyWaitSec);

				if(response.statusCode == 200)
					continue;
			}
			catch(std::exception& e) { }

			notReadyServiceHost = remote.host + ":" + std::to_string(remote.port);
			break;
		}

		if(notReadyServiceHost.empty() )
			return;

		if(Clock::now() >= endWaitT)
			throw ProgError("Timed out waiting for services to become ready. "
				"Unreachable service: " + notReadyServiceHost);

		usleep(1000 * 1000);
	}
}

/* expected entries / bytes of all services together, for the "Done%" column of the live CSV */
void Master::getExpectedTotals(int benchPhase, uint64_t& outEntries, uint64_t& outBytes)
{
	outEntries = outBytes = 0;

	try
	{
		ProgArgs::ABIConfig abiConfig;
		progArgs.toABIConfig(abiConfig);

		if(abiConfig.gpuIDs.empty() )
		{
			abiConfig.gpuIDs.push_back(0);
			abiConfig.cfg.gpuIDs = abiConfig.gpuIDs.data();
			abiConfig.cfg.numGPUIDs = 1;
		}

		abiConfig.cfg.pathType = progArgs.benchPathType; // (as reported by the services)
		abiConfig.cfg.treeFilePath = NULL;
		abiConfig.cfg.numDataSetThreads = (uint32_t)(progArgs.noSharedServicePath ?
			progArgs.numThreads : (progArgs.numThreads * hosts.size() ) );

		const Config cfg = Config::fromABI(&abiConfig.cfg);
		uint64_t entriesPerWorker, bytesPerWorker;

		expectedPerWorker(cfg, benchPhase, entriesPerWorker, bytesPerWorker);

		outEntries = entriesPerWorker * progArgs.numThreads * hosts.size();
		outBytes = bytesPerWorker * progArgs.numThreads * hosts.size();
	}
	catch(std::exception& e) { }
}

/* Statistics::printLiveStatsCSV in a distributed run (Statistics.cpp:3017-3230): a "Total" line
 * per update (plus a "Read" line in rwmix phases) and, with --livecsvex, one line per service
 * with its threads left, CPU utilisation and host name */
void Master::printLiveStatsCSV(int benchPhase, elb_liveops oldLiveOps[2], Clock::time_point& lastT,
	const Clock::time_point& phaseStartT, uint64_t expectedEntries, uint64_t expectedBytes)
{
	const bool toStdout = (progArgs.liveCSVFilePath == "stdout");
	std::ofstream fileStream;
	bool printHeaders = toStdout ? !liveCSVHeaderPrinted : false;

	if(!toStdout)
	{
		struct stat statBuf;
		printHeaders = (stat(progArgs.liveCSVFilePath.c_str(), &statBuf) != 0) ||
			!statBuf.st_size;

		fileStream.open(progArgs.liveCSVFilePath, std::ofstream::app);

		if(!fileStream)
			throw ProgError("Unable to open live stats csv file: " + progArgs.liveCSVFilePath);
	}

	std::ostream& out = toStdout ? std::cout : fileStream;

	if(printHeaders)
		out << "ISO Date,Label,Phase,RuntimeMS,Rank,MixType,Done%,DoneBytes,MiB/s,IOPS,Entries,"
			"Entries/s,Lat Ent us,Lat IO us,Active,CPU,Service," << std::endl;

	liveCSVHeaderPrinted = true;

	elb_liveops liveOps[2] = {};
	elb_livelat liveLat = {};
	uint64_t numThreadsLeft = 0, cpuSum = 0;

	for(RemoteHost& remote : hosts)
	{
		liveOpsAdd(liveOps[0], remote.liveOps);
		liveOpsAdd(liveOps[1], remote.liveOpsReadMix);
		liveLat.numAvgIOLatValues += remote.liveLat.numAvgIOLatValues;
		liveLat.avgIOLatMicroSecsSum += remote.liveLat.avgIOLatMicroSecsSum;
		liveLat.numAvgEntriesLatValues += remote.liveLat.numAvgEntriesLatValues;
		liveLat.avgEntriesLatMicroSecsSum += remote.liveLat.avgEntriesLatMicroSecsSum;
		remote.liveLat = elb_livelat{};
		numThreadsLeft += progArgs.numThreads - std::min(progArgs.numThreads,
			(uint64_t)remote.numWorkersDone);
		cpuSum += remote.cpuUtilLive;
	}

	const Clock::time_point nowT = Clock::now();
	const uint64_t intervalUSec =
		std::chrono::duration_cast<std::chrono::microseconds>(nowT - lastT).count();
	const uint64_t elapsedMS =
		std::chrono::duration_cast<std::chrono::milliseconds>(nowT - phaseStartT).count();
	const bool isRWMixPhase = (liveOps[1].numBytesDone || liveOps[1].numEntriesDone);
	const bool isDirMode = (progArgs.benchPathType == ELB_PATH_DIR);
	const std::string phaseName = stats::phaseName(benchPhase, progArgs);
	std::string label = progArgs.benchLabel;
	std::replace(label.begin(), label.end(), ',', ' ');

	char isoBuf[64];
	{
		struct timeval timeVal;
		gettimeofday(&timeVal, NULL);
		struct tm localTimeInfo;
		localtime_r(&timeVal.tv_sec, &localTimeInfo);
		char dateBuf[32], zoneBuf[16];
		strftime(dateBuf, sizeof(dateBuf), "%FT%T", &localTimeInfo);
		strftime(zoneBuf, sizeof(zoneBuf), "%z", &localTimeInfo);
		snprintf(isoBuf, sizeof(isoBuf), "%s.%03d%s", dateBuf, (int)(timeVal.tv_usec / 1000),
			zoneBuf);
	}

	auto perSec = [&](uint64_t newVal, uint64_t oldVal)
		{ return intervalUSec ? perSecFromUSec(newVal - oldVal, intervalUSec) : 0; };
	auto percentDone = [](const elb_liveops& ops, uint64_t bytesTotal, uint64_t entriesTotal)
	{
		uint64_t percent = 0;

		if(bytesTotal)
			percent = (100 * ops.numBytesDone) / bytesTotal;
		else
		if(entriesTotal)
			percent = (100 * ops.numEntriesDone) / entriesTotal;

		return std::min(percent, (uint64_t)100);
	};
	auto avg = [](uint64_t sum, uint64_t num) { return num ? (sum / num) : 0; };

	for(int mixIdx = 0; mixIdx < (isRWMixPhase ? 2 : 1); mixIdx++)
	{
		const elb_liveops& ops = liveOps[mixIdx];

		out << isoBuf << "," << label << "," << phaseName << "," << elapsedMS << "," <<
			"Total" << "," << (isRWMixPhase ? (mixIdx ? "Read" : "Write") : "") << "," <<
			percentDone(ops, expectedBytes, expectedEntries) << "," << ops.numBytesDone << "," <<
			(perSec(ops.numBytesDone, oldLiveOps[mixIdx].numBytesDone) / (1024 * 1024) ) << "," <<
			perSec(ops.numIOPSDone, oldLiveOps[mixIdx].numIOPSDone) << "," <<
			(isDirMode ? ops.numEntriesDone : 0) << "," <<
			(isDirMode ? perSec(ops.numEntriesDone, oldLiveOps[mixIdx].numEntriesDone) : 0) <<
			"," << (mixIdx ? 0 : avg(liveLat.avgEntriesLatMicroSecsSum,
				liveLat.numAvgEntriesLatValues) ) << "," <<
			(mixIdx ? 0 : avg(liveLat.avgIOLatMicroSecsSum, liveLat.numAvgIOLatValues) ) << "," <<
			numThreadsLeft << "," << (hosts.empty() ? 0 : (cpuSum / hosts.size() ) ) << "," <<
			"" << "," << std::endl;

		oldLiveOps[mixIdx] = ops;
	}

	lastT = nowT;

	if(!progArgs.useExtendedLiveCSV)
		return;

	for(size_t hostIdx = 0; hostIdx < hosts.size(); hostIdx++)
	{
		const RemoteHost& remote = hosts[hostIdx];
		const elb_liveops remoteOps[2] = {remote.liveOps, remote.liveOpsReadMix};

		for(int mixIdx = 0; mixIdx < (isRWMixPhase ? 2 : 1); mixIdx++)
			out << isoBuf << "," << label << "," << phaseName << "," << elapsedMS << "," <<
				hostIdx << "," << (isRWMixPhase ? (mixIdx ? "Read" : "Write") : "") << "," <<
				percentDone(remoteOps[mixIdx], expectedBytes / hosts.size(),
					expectedEntries / hosts.size() ) << "," <<
				remoteOps[mixIdx].numBytesDone << "," << "" << "," << "" << "," <<
				(isDirMode ? remoteOps[mixIdx].numEntriesDone : 0) << "," << "" << "," << "" <<
				"," << "" << "," <<
				(progArgs.numThreads - std::min(progArgs.numThreads,
					(uint64_t)remote.numWorkersDone) ) << "," << remote.cpuUtilLive << "," <<
				remote.host << ":" << remote.port << "," << std::endl;
	}
}

/* Coordinator::rotateHosts (Coordinator.cpp:382-404) + ProgArgs::rotateHosts (:4137-4144): between
 * phases the services swap ranks, which needs a new preparation phase on all of them */
void Master::rotateHosts()
{
	if( (hosts.size() < 2) || !progArgs.rotateHostsNum)
		return;

	interruptAll(false);

	for(uint64_t i = 0; i < progArgs.rotateHostsNum; i++)
		std::rotate(hosts.begin(), hosts.begin() + 1, hosts.end() );

	prepareRemotePhases();
}

int Master::run()
{
	initHosts();

	try
	{
		waitForServicesReady();

		prepareRemotePhases();

		waitForUserDefinedStartTime(progArgs);

		struct BenchPhaseConfig { int benchPhase; bool runPhase; };

		const BenchPhaseConfig allBenchPhases[] =
		{
			{ELB_PHASE_CREATEDIRS, progArgs.runCreateDirsPhase},
			{ELB_PHASE_CREATEFILES, progArgs.runCreateFilesPhase},
			{ELB_PHASE_STATFILES, progArgs.runStatFilesPhase},
			{ELB_PHASE_READFILES, progArgs.runReadPhase},
			{ELB_PHASE_DELETEFILES, progArgs.runDeleteFilesPhase},
			{ELB_PHASE_DELETEDIRS, progArgs.runDeleteDirsPhase},
		};

		for(uint64_t iterationIndex = 0; iterationIndex < progArgs.iterations; iterationIndex++)
		{
			if(progArgs.iterations > 1)
				std::cout << "[Starting iteration " << (iterationIndex + 1) << " of " <<
					progArgs.iterations << "...]" << std::endl;

			stats::printPhaseResultsTableHeader(std::cout);

			runSyncAndDropCaches();

			bool isFirstPhase = true;

			for(const BenchPhaseConfig& phaseConfig : allBenchPhases)
			{
				if(!phaseConfig.runPhase)
					continue;

				if(!isFirstPhase)
					rotateHosts();

				isFirstPhase = false;

				runPhase(phaseConfig.benchPhase);
				runSyncAndDropCaches();
			}
		}
	}
	catch(ProgTimeLimit& e)
	{ // a user-defined time limit, not an error
		std::cout << e.what() << std::endl;
	}
	catch(std::exception& e)
	{
		std::cerr << "ERROR: " << e.what() << std::endl;
		interruptAll(false);
		return EXIT_FAILURE;
	}

	interruptAll(false); // release the services' resources (RemoteWorker::interruptBenchPhase)

	return EXIT_SUCCESS;
}

int Master::interruptOrQuit()
{
	initHosts();
	interruptAll(progArgs.quitServices);
	return EXIT_SUCCESS;
}

int masterMain(ProgArgs& progArgs)
{
	Master master(progArgs);
	return master.run();
}

int masterInterruptOrQuitServices(ProgArgs& progArgs)
{
	Master master(progArgs);
	return master.interruptOrQuit();
}

} // namespace elb
